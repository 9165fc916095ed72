// Per-warp rigid-body engine: one environment per warp, state in shared memory, lanes split bodies / dofs /
// matrix entries / constraint rows.  Smooth dynamics part: kinematics, body velocities, RNE bias, passive + fluid
// forces, composite inertia -> M, actuation, Euler integration.
//
// Replaces the engine work behind MjSim.step1/step2 (robosuite/utils/binding_utils.py:1101-1107) - SURVEY.md
// section 8 rows a1 and a7.  Spatial quantities are expressed about the world origin in world axes.
#pragma once
#include "b2s_math.cuh"


// ------------------------------------------------------------------------------------------- small SPD solve
// x <- (A + diag(hd))^-1 x for an n x n symmetric positive definite A (n <= NVP <= 32), A and x in shared memory.
// Lane i keeps the FULL row i of the symmetric working matrix in registers: at elimination step j lane j's row is
// column j of L (by symmetry), so the rank-1 update needs one shuffle + one FMA per entry and both triangular solves
// read only the lane's own registers.  Returns non-zero (warp-uniform) if a pivot was not positive.
template <typename R> DEV R r_rsqrt(R x);
template <> DEV float r_rsqrt<float>(float x) { float y = rsqrtf(x); return y * (1.5f - 0.5f * x * y * y); }
template <> DEV double r_rsqrt<double>(double x) { return 1.0 / sqrt(x); }

template <typename R, int NVP>
DEVN int spd_solve_reg(const R* A, int n, const R* dadd, R dscale, R* x, int lane) {
  R a[NVP];  // must stay in registers: every index below is a compile-time constant after unrolling
  int row = lane < n ? lane : 0;
  R dl = (dadd != nullptr && lane < n) ? dscale * dadd[row] : R(0);
#pragma unroll
  for (int k = 0; k < NVP; k++) {
    R v = (k < n) ? A[row * n + (k < n ? k : 0)] : R(0);
    v = lane < n ? v : R(0);
    a[k] = v + ((k == lane) ? (lane < n ? dl : R(1)) : R(0));
  }
  R b = lane < n ? x[row] : R(0);
  R invd = 1;  // 1 / L[lane][lane]
  int bad = 0;
  // After step j: lanes i > j hold l_ij in a[j]; lane j keeps its row entries a[k], k > j, UNSCALED (u_jk = a[k] * invd is
  // formed where it is used), which leaves one multiply + shuffle + FMA per trailing entry and no selects.
#pragma unroll
  for (int j = 0; j < NVP; j++) {
    R d = __shfl_sync(B2S_FULL, a[j], j);
    if (!(d > Lim<R>::minval())) { bad = 1; d = Lim<R>::minval(); }
    R inv = r_rsqrt(d);
    invd = (lane == j) ? inv : invd;
    R lj = (lane > j) ? a[j] * inv : R(0);
    a[j] = (lane > j) ? lj : a[j];
#pragma unroll
    for (int k = j + 1; k < NVP; k++) {
      R u = __shfl_sync(B2S_FULL, a[k], j) * inv;  // l_kj
      a[k] -= lj * u;
    }
  }
  // forward: L y = b
#pragma unroll
  for (int k = 0; k < NVP; k++) {
    R yk = __shfl_sync(B2S_FULL, b * invd, k);
    R t = (lane > k) ? a[k] : R(0);
    b = (lane == k) ? yk : b - t * yk;
  }
  // backward: L^T x = y   (u_lane,k = a[k] * invd for k > lane)
#pragma unroll
  for (int k = NVP - 1; k >= 0; k--) {
    R xk = __shfl_sync(B2S_FULL, b * invd, k);
    R t = (lane < k) ? a[k] * invd : R(0);
    b = (lane == k) ? xk : b - t * xk;
  }
  if (lane < n) x[lane] = b;
  __syncwarp();
  return bad;
}

// Block-diagonal variant: the matrix couples dofs only within kinematic trees (always true for M and M + h D, true for
// the Newton Hessian when no active contact joins two different moving trees).  Every tree is eliminated at the same
// time by its own lanes: lane i keeps row i restricted to its tree's columns (NVB = padded size of the largest tree).
// Lanes whose tree is smaller than the current column see d = 1, l = 0 and shuffle from themselves: no-ops without selects.
template <typename R, int NVB>
DEVN int spd_solve_blk(const R* A, int n, const R* dadd, R dscale, R* x, int lane, const int* dof_treebase, const int* dof_treesize) {
  R a[NVB];
  int row = lane < n ? lane : 0;
  int base = dof_treebase[row], size = dof_treesize[row];
  int li = row - base;  // local index of this lane's row inside its tree
  if (lane >= n) size = 0;
  R dl = (dadd != nullptr && lane < n) ? dscale * dadd[row] : R(0);
#pragma unroll
  for (int k = 0; k < NVB; k++) {
    R v = (k < size) ? A[row * n + base + (k < size ? k : 0)] : R(0);
    a[k] = v + ((k == li && lane < n) ? dl : R(0));
  }
  R b = lane < n ? x[row] : R(0);
  R invd = 1;
  int bad = 0;
#pragma unroll
  for (int j = 0; j < NVB; j++) {
    bool on = j < size;
    int src = on ? base + j : lane;
    R d = __shfl_sync(B2S_FULL, a[j], src);
    if (on && !(d > Lim<R>::minval())) { bad = 1; d = Lim<R>::minval(); }
    if (!on) d = 1;
    R inv = r_rsqrt(d);
    invd = (on && li == j) ? inv : invd;
    R lj = (on && li > j) ? a[j] * inv : R(0);
    a[j] = (on && li > j) ? lj : a[j];
#pragma unroll
    for (int k = j + 1; k < NVB; k++) {
      R u = __shfl_sync(B2S_FULL, a[k], src) * inv;
      a[k] -= lj * u;
    }
  }
#pragma unroll
  for (int k = 0; k < NVB; k++) {
    bool on = k < size;
    R yk = __shfl_sync(B2S_FULL, b * invd, on ? base + k : lane);
    R t = (on && li > k) ? a[k] : R(0);
    b = (on && li == k) ? yk : b - t * yk;
  }
#pragma unroll
  for (int k = NVB - 1; k >= 0; k--) {
    bool on = k < size;
    R xk = __shfl_sync(B2S_FULL, b * invd, on ? base + k : lane);
    R t = (on && li < k) ? a[k] * invd : R(0);
    b = (on && li == k) ? xk : b - t * xk;
  }
  if (lane < n) x[lane] = b;
  __syncwarp();
  return __any_sync(B2S_FULL, bad);
}

// ---- per-environment model values (b2s_model_override): the environment's override where one is declared, the model's value
// otherwise.  A handle without overrides pays the test of n_mg / n_mb / a null pointer, uniform across the warp.
template <typename R> DEV const R* geom_size_of(const DModel<R>& m, const DState<R>& s, int g, int env) {
  for (int k = 0; k < s.n_mg; k++) if (s.mg_id[k] == g) return s.mg_size + 3 * ((size_t)k * s.n_env + env);
  return m.geom_size + 3 * g;
}
template <typename R> DEV const R* geom_friction_of(const DModel<R>& m, const DState<R>& s, int g, int env) {
  for (int k = 0; k < s.n_mg; k++) if (s.mg_id[k] == g) return s.mg_fric + 3 * ((size_t)k * s.n_env + env);
  return m.geom_friction + 3 * g;
}
template <typename R> DEV R geom_rbound_of(const DModel<R>& m, const DState<R>& s, int g, int env) {
  for (int k = 0; k < s.n_mg; k++) if (s.mg_id[k] == g) return s.mg_rbound[(size_t)k * s.n_env + env];
  return m.geom_rbound[g];
}
template <typename R> DEV const R* geom_aabb_of(const DModel<R>& m, const DState<R>& s, int g, int env) {
  for (int k = 0; k < s.n_mg; k++) if (s.mg_id[k] == g) return s.mg_aabb + 6 * ((size_t)k * s.n_env + env);
  return m.geom_aabb + 6 * g;
}
template <typename R> DEV R body_mass_of(const DModel<R>& m, const DState<R>& s, int b, int env) {
  for (int k = 0; k < s.n_mb; k++) if (s.mb_id[k] == b) return s.mb_mass[(size_t)k * s.n_env + env];
  return m.body_mass[b];
}
template <typename R> DEV const R* body_inertia_of(const DModel<R>& m, const DState<R>& s, int b, int env) {
  for (int k = 0; k < s.n_mb; k++) if (s.mb_id[k] == b) return s.mb_inertia + 3 * ((size_t)k * s.n_env + env);
  return m.body_inertia + 3 * b;
}
template <typename R> DEV const R* geom_solref_of(const DModel<R>& m, const DState<R>& s, int g, int env) {
  for (int k = 0; k < s.n_mg; k++) if (s.mg_id[k] == g) return s.mg_solref + 2 * ((size_t)k * s.n_env + env);
  return m.geom_solref + 2 * g;
}
template <typename R> DEV const R* geom_solimp_of(const DModel<R>& m, const DState<R>& s, int g, int env) {
  for (int k = 0; k < s.n_mg; k++) if (s.mg_id[k] == g) return s.mg_solimp + 5 * ((size_t)k * s.n_env + env);
  return m.geom_solimp + 5 * g;
}
// whole dof vectors: a stage picks the row once, at its top, and its loops index it (no lookup inside the arithmetic)
template <typename R> DEV const R* dof_damping_of(const DModel<R>& m, const DState<R>& s, int env) {
  return s.dof_damp ? s.dof_damp + (size_t)env * m.nv : m.dof_damping;
}
template <typename R> DEV const R* dof_armature_of(const DModel<R>& m, const DState<R>& s, int env) {
  return s.dof_arm ? s.dof_arm + (size_t)env * m.nv : m.dof_armature;
}
template <typename R> DEV const R* dof_frictionloss_of(const DModel<R>& m, const DState<R>& s, int env) {
  return s.dof_floss ? s.dof_floss + (size_t)env * m.nv : m.dof_frictionloss;
}
// constants derived at qpos0 (the set-constants pass writes them per environment once a handle declares an override)
template <typename R> DEV const R* dof_invweight0_of(const DModel<R>& m, const DState<R>& s, int env) {
  return s.dof_iw ? s.dof_iw + (size_t)env * m.nv : m.dof_invweight0;
}
template <typename R> DEV const R* body_invweight0_of(const DModel<R>& m, const DState<R>& s, int env) {
  return s.body_iw ? s.body_iw + (size_t)env * 2 * m.nbody : m.body_invweight0;
}
template <typename R> DEV R meaninertia_of(const DModel<R>& m, const DState<R>& s, int env) {
  return s.mean_inertia ? s.mean_inertia[env] : m.meaninertia;
}

template <typename R>
struct Eng {
  R* ws;  // this warp's workspace
  int lane;
  int slot, lid;  // descriptor slot of the owning handle, workspace layout of the running kernel (LAY_*)
  int env = 0;    // environment index (per-environment poses of world-welded bodies and model overrides): set by every stage that
                  // starts an environment (kinematics, the tail's rows)

  DEV Eng(R* ws_, int lane_, int slot_, int lid_) : ws(ws_), lane(lane_), slot(slot_), lid(lid_) {}
  DEV const DModel<R>& model() const { return cmodel<R>(slot); }
  DEV const DState<R>& state() const { return cstate<R>(slot); }
  DEV const WSLayout& lay() const { return c_lay[slot][lid]; }
  DEV const CtrlCfgDev& ccfg() const { return c_cc[slot]; }
  DEV R* p(int off) const { return ws + off; }
  DEV int* pi(int off) const { return reinterpret_cast<int*>(ws + off); }

  // ------------------------------------------------------------------------------------------- kinematics
  // mj_checkPos / mj_checkVel / mj_checkAcc of the reference engine (the first calls of mj_step, and after the solve): a non-finite
  // or huge (> 1e10) coordinate means the simulation diverged; the engine warns and resets the data to the model defaults instead
  // of integrating garbage (which here would also run every solver loop to its iteration cap).  Warp-uniform result.
  DEV int vec_bad(const R* x, int n) const {
    int b = 0;
    for (int i = lane; i < n; i += 32) b |= !(r_abs(x[i]) <= R(1e10));
    return warp_or_i(b);
  }
  // returns 32 when the state was reset (callers clear the rest of the per-environment data: acceleration, warm start, time)
  DEVN int kinematics() {
    const DModel<R>& m = model(); const WSLayout& L = lay();
    R* xpos = p(L.xpos); R* xquat = p(L.xquat); R* xmat = p(L.xmat);
    int was_reset = 0;
    if (vec_bad(p(L.qpos), m.nq) | vec_bad(p(L.qvel), m.nv)) {
      for (int i = lane; i < m.nq; i += 32) p(L.qpos)[i] = m.qpos0[i];
      for (int i = lane; i < m.nv; i += 32) p(L.qvel)[i] = 0;
      was_reset = 32;
      __syncwarp();
    }
    const R* qpos = p(L.qpos);
    // bodies welded to the world: constant pose, the environment's override, or (tree overrides) the override of the root they
    // follow composed with their fixed pose relative to it
    for (int b = lane; b < m.nbody; b += 32)
      if (m.body_weldid[b] == 0) {
        const R* px = m.body_xpos0 + 3 * b; const R* pq = m.body_xquat0 + 4 * b;
        const DState<R>& st = state();
        for (int k = 0; k < st.n_ov; k++)
          if (st.ov_body[k] == b) { px = st.ov_pos[k] + 3 * (size_t)env; pq = st.ov_quat[k] + 4 * (size_t)env; }
        R tp[3], tq[4];
        const int root = st.ov_tree ? st.ov_tree[b] : -1;
        if (root >= 0) {
          const R* rp = st.ov_pos[root] + 3 * (size_t)env; const R* rq = st.ov_quat[root] + 4 * (size_t)env;
          const R* rel = st.ov_rel + 7 * b;
          qrot(tp, rq, rel);
          tp[0] += rp[0]; tp[1] += rp[1]; tp[2] += rp[2];
          qmul(tq, rq, rel + 3);
          px = tp; pq = tq;
        }
        R q[4] = {pq[0], pq[1], pq[2], pq[3]};
        xpos[3 * b] = px[0]; xpos[3 * b + 1] = px[1]; xpos[3 * b + 2] = px[2];
        xquat[4 * b] = q[0]; xquat[4 * b + 1] = q[1]; xquat[4 * b + 2] = q[2]; xquat[4 * b + 3] = q[3];
        q2mat(xmat + 9 * b, q);
      }
    __syncwarp();
    // moving bodies.  (1) every body in parallel: its pose relative to the parent frame (lp, lq) including the joint
    // displacement; (2) one tree level at a time, the short serial part: compose with the finished parent pose;
    // (3) rotation matrices of all bodies in parallel.
    R* loc = p(L.scratch);  // 8 words per body: lp[3], lq[4], absolute flag (free joints give world poses directly)
    for (int b = lane; b < m.nbody; b += 32) {
      if (m.body_weldid[b] == 0) continue;
      R lp[3] = {m.body_pos[3 * b], m.body_pos[3 * b + 1], m.body_pos[3 * b + 2]};
      R lq[4] = {m.body_quat[4 * b], m.body_quat[4 * b + 1], m.body_quat[4 * b + 2], m.body_quat[4 * b + 3]};
      R absolute = 0;
      int j = m.body_jntid[b];
      if (j >= 0) {
        int t = m.jnt_type[j], qa = m.jnt_qposadr[j];
        if (t == JNT_FREE) {
          lp[0] = qpos[qa]; lp[1] = qpos[qa + 1]; lp[2] = qpos[qa + 2];
          lq[0] = qpos[qa + 3]; lq[1] = qpos[qa + 4]; lq[2] = qpos[qa + 5]; lq[3] = qpos[qa + 6];
          absolute = 1;
        } else {
          R ax[3] = {m.jnt_axis[3 * j], m.jnt_axis[3 * j + 1], m.jnt_axis[3 * j + 2]};
          R dq = qpos[qa] - m.qpos0[qa];
          if (t == JNT_SLIDE) {
            R axp[3];
            qrot(axp, lq, ax);
            v3addscl(lp, lp, axp, dq);
          } else {  // hinge: rotate about the joint anchor (anchor = lp + R(body_quat) jnt_pos stays fixed)
            R jp[3] = {m.jnt_pos[3 * j], m.jnt_pos[3 * j + 1], m.jnt_pos[3 * j + 2]};
            R a0[3], a1[3], ql[4], qn[4];
            qrot(a0, lq, jp);
            aa2quat(ql, ax, dq);
            qmul(qn, lq, ql);
            qrot(a1, qn, jp);
            lp[0] += a0[0] - a1[0]; lp[1] += a0[1] - a1[1]; lp[2] += a0[2] - a1[2];
            lq[0] = qn[0]; lq[1] = qn[1]; lq[2] = qn[2]; lq[3] = qn[3];
          }
        }
      }
      R* o = loc + 8 * b;
      o[0] = lp[0]; o[1] = lp[1]; o[2] = lp[2]; o[3] = lq[0]; o[4] = lq[1]; o[5] = lq[2]; o[6] = lq[3]; o[7] = absolute;
    }
    __syncwarp();
    for (int lev = 1; lev <= m.maxdepth; lev++) {
      for (int b = lane; b < m.nbody; b += 32) {
        if (m.body_depth[b] != lev || m.body_weldid[b] == 0) continue;
        const R* o = loc + 8 * b;
        R pos[3] = {o[0], o[1], o[2]}, quat[4] = {o[3], o[4], o[5], o[6]};
        if (o[7] == R(0)) {
          int par = m.body_parentid[b];
          R t[3];
          qrot(t, xquat + 4 * par, pos);
          v3add(pos, t, xpos + 3 * par);
          R lq[4] = {quat[0], quat[1], quat[2], quat[3]};
          qmul(quat, xquat + 4 * par, lq);
        }
        qnormalize(quat);
        xpos[3 * b] = pos[0]; xpos[3 * b + 1] = pos[1]; xpos[3 * b + 2] = pos[2];
        xquat[4 * b] = quat[0]; xquat[4 * b + 1] = quat[1]; xquat[4 * b + 2] = quat[2]; xquat[4 * b + 3] = quat[3];
      }
      __syncwarp();
    }
    for (int b = lane; b < m.nbody; b += 32)
      if (m.body_weldid[b] != 0) q2mat(xmat + 9 * b, xquat + 4 * b);
    __syncwarp();
    // per body: inertial frame origin + spatial inertia about the world origin
    R* xipos = p(L.xipos); R* cinert = p(L.cinert);
    for (int b = lane; b < m.nbody; b += 32) {
      // the override lookups come first: the arithmetic below stays in one basic block, where nvcc forms the same FMAs as without them
      const R* bi = body_inertia_of(m, state(), b, env);
      const R mass = body_mass_of(m, state(), b, env);
      R ip[3] = {m.body_ipos[3 * b], m.body_ipos[3 * b + 1], m.body_ipos[3 * b + 2]};
      R c[3], qi[4], Ri[9];
      m3mulv(c, xmat + 9 * b, ip);
      v3add(c, c, xpos + 3 * b);
      xipos[3 * b] = c[0]; xipos[3 * b + 1] = c[1]; xipos[3 * b + 2] = c[2];
      R iq[4] = {m.body_iquat[4 * b], m.body_iquat[4 * b + 1], m.body_iquat[4 * b + 2], m.body_iquat[4 * b + 3]};
      qmul(qi, xquat + 4 * b, iq);
      q2mat(Ri, qi);
      R I0 = bi[0], I1 = bi[1], I2 = bi[2];
      R* ci = cinert + 10 * b;
      R cc = v3dot(c, c);
#define IW(r, s) (Ri[3 * r] * I0 * Ri[3 * s] + Ri[3 * r + 1] * I1 * Ri[3 * s + 1] + Ri[3 * r + 2] * I2 * Ri[3 * s + 2])
      ci[0] = IW(0, 0) + mass * (cc - c[0] * c[0]);
      ci[1] = IW(1, 1) + mass * (cc - c[1] * c[1]);
      ci[2] = IW(2, 2) + mass * (cc - c[2] * c[2]);
      ci[3] = IW(0, 1) - mass * c[0] * c[1];
      ci[4] = IW(0, 2) - mass * c[0] * c[2];
      ci[5] = IW(1, 2) - mass * c[1] * c[2];
#undef IW
      ci[6] = mass * c[0]; ci[7] = mass * c[1]; ci[8] = mass * c[2]; ci[9] = mass;
    }
    // per dof: spatial motion axis
    R* cdof = p(L.cdof);
    for (int i = lane; i < m.nv; i += 32) {
      int j = m.dof_jntid[i], b = m.dof_bodyid[i], kind = m.dof_kind[i], k = i - m.jnt_dofadr[j];
      R* c = cdof + 6 * i;
      const R* Rb = xmat + 9 * b;
      if (kind == DK_FREE_T) {
        c[0] = c[1] = c[2] = 0; c[3] = k == 0; c[4] = k == 1; c[5] = k == 2;
      } else if (kind == DK_FREE_R) {
        int col = k - 3;
        R w[3] = {Rb[col], Rb[3 + col], Rb[6 + col]};
        c[0] = w[0]; c[1] = w[1]; c[2] = w[2];
        v3cross(c + 3, xpos + 3 * b, w);
      } else {
        R ax[3] = {m.jnt_axis[3 * j], m.jnt_axis[3 * j + 1], m.jnt_axis[3 * j + 2]}, axw[3];
        m3mulv(axw, Rb, ax);
        if (kind == DK_SLIDE) { c[0] = c[1] = c[2] = 0; c[3] = axw[0]; c[4] = axw[1]; c[5] = axw[2]; }
        else {
          R jp[3] = {m.jnt_pos[3 * j], m.jnt_pos[3 * j + 1], m.jnt_pos[3 * j + 2]}, anchor[3];
          m3mulv(anchor, Rb, jp);
          v3add(anchor, anchor, xpos + 3 * b);
          c[0] = axw[0]; c[1] = axw[1]; c[2] = axw[2];
          v3cross(c + 3, anchor, axw);
        }
      }
    }
    // colliding geoms and sites
    R* gpos = p(L.gpos); R* gmat = p(L.gmat);
    for (int k = lane; k < m.ncg; k += 32) {
      int g = m.cg_geom[k], b = m.geom_bodyid[g];
      R gp[3] = {m.geom_pos[3 * g], m.geom_pos[3 * g + 1], m.geom_pos[3 * g + 2]}, t[3], q[4];
      R gq[4] = {m.geom_quat[4 * g], m.geom_quat[4 * g + 1], m.geom_quat[4 * g + 2], m.geom_quat[4 * g + 3]};
      m3mulv(t, xmat + 9 * b, gp);
      v3add(gpos + 3 * k, t, xpos + 3 * b);
      qmul(q, xquat + 4 * b, gq);
      q2mat(gmat + 9 * k, q);
    }
    R* spos = p(L.spos); R* smat = p(L.smat);
    for (int s = lane; s < m.nsite; s += 32) {
      int b = m.site_bodyid[s];
      R sp[3] = {m.site_pos[3 * s], m.site_pos[3 * s + 1], m.site_pos[3 * s + 2]}, t[3], q[4];
      R sq[4] = {m.site_quat[4 * s], m.site_quat[4 * s + 1], m.site_quat[4 * s + 2], m.site_quat[4 * s + 3]};
      m3mulv(t, xmat + 9 * b, sp);
      v3add(spos + 3 * s, t, xpos + 3 * b);
      qmul(q, xquat + 4 * b, sq);
      q2mat(smat + 9 * s, q);
    }
    __syncwarp();
    return was_reset;
  }

  // last dof on the kinematic chain ending at body b (-1 if none)
  DEV int chain_end(int b) const {
    const DModel<R>& m = model();
    while (b > 0 && m.body_dofnum[b] == 0) b = m.body_parentid[b];
    return b > 0 ? m.body_dofadr[b] + m.body_dofnum[b] - 1 : -1;
  }

  // ------------------------------------------------------------------------------------------- velocity stage
  // cvel, cdof_dot, RNE bias forces, passive (damping + fluid + joint spring) forces
  DEVN void velocity() {
    const DModel<R>& m = model(); const WSLayout& L = lay();
    const R* cdof = p(L.cdof); const R* qvel = p(L.qvel);
    R* cvel = p(L.cvel); R* cdd = p(L.cdofdot);
    for (int b = lane; b < m.nbody; b += 32) {
      R v[6] = {0, 0, 0, 0, 0, 0};
      for (int i = chain_end(b); i >= 0; i = m.dof_parentid[i]) {
        R qv = qvel[i];
#pragma unroll
        for (int e = 0; e < 6; e++) v[e] += cdof[6 * i + e] * qv;
      }
#pragma unroll
      for (int e = 0; e < 6; e++) cvel[6 * b + e] = v[e];
    }
    // cdof_dot = (velocity accumulated before this dof) x cdof
    for (int i = lane; i < m.nv; i += 32) {
      R* o = cdd + 6 * i;
      if (m.dof_kind[i] == DK_FREE_T) { o[0] = o[1] = o[2] = o[3] = o[4] = o[5] = 0; continue; }
      R v[6] = {0, 0, 0, 0, 0, 0};
      for (int a = m.dof_cddstart[i]; a >= 0; a = m.dof_parentid[a]) {
        R qv = qvel[a];
#pragma unroll
        for (int e = 0; e < 6; e++) v[e] += cdof[6 * a + e] * qv;
      }
      cross_motion(o, v, cdof + 6 * i);
    }
    __syncwarp();
    // per body: acceleration bias, inertial force, fluid force
    R* frne = p(L.frne); R* ffl = p(L.ffl);
    const R* cinert = p(L.cinert); const R* xipos = p(L.xipos); const R* xquat = p(L.xquat);
    for (int b = lane; b < m.nbody; b += 32) {
      R a[6] = {0, 0, 0, -m.gravity[0], -m.gravity[1], -m.gravity[2]};
      for (int i = chain_end(b); i >= 0; i = m.dof_parentid[i]) {
        R qv = qvel[i];
#pragma unroll
        for (int e = 0; e < 6; e++) a[e] += cdd[6 * i + e] * qv;
      }
      R Ia[6], Iv[6], x[6];
      inert_mulv(Ia, cinert + 10 * b, a);
      inert_mulv(Iv, cinert + 10 * b, cvel + 6 * b);
      cross_force(x, cvel + 6 * b, Iv);
      if (b == 0) {
#pragma unroll
        for (int e = 0; e < 6; e++) { Ia[e] = 0; x[e] = 0; }
      }
#pragma unroll
      for (int e = 0; e < 6; e++) frne[6 * b + e] = Ia[e] + x[e];
      // fluid (inertia-box model); result as spatial force about the world origin
      R ff[6] = {0, 0, 0, 0, 0, 0};
      R mass = body_mass_of(m, state(), b, env);
      if (b > 0 && mass >= Lim<R>::minval() && (m.density > 0 || m.viscosity > 0)) {
        const R* bi = body_inertia_of(m, state(), b, env);
        R I0 = bi[0], I1 = bi[1], I2 = bi[2];
        R box[3];
        box[0] = r_sqrt(r_max(Lim<R>::minval(), I1 + I2 - I0) / mass * R(6));
        box[1] = r_sqrt(r_max(Lim<R>::minval(), I0 + I2 - I1) / mass * R(6));
        box[2] = r_sqrt(r_max(Lim<R>::minval(), I0 + I1 - I2) / mass * R(6));
        R qi[4], Ri[9], iq[4] = {m.body_iquat[4 * b], m.body_iquat[4 * b + 1], m.body_iquat[4 * b + 2], m.body_iquat[4 * b + 3]};
        qmul(qi, xquat + 4 * b, iq);
        q2mat(Ri, qi);
        const R* cv = cvel + 6 * b;
        const R* c = xipos + 3 * b;
        R lin[3], t[3], lv[6], lf[6] = {0, 0, 0, 0, 0, 0};
        v3cross(t, cv, c);
        v3add(lin, cv + 3, t);
        lin[0] -= m.wind[0]; lin[1] -= m.wind[1]; lin[2] -= m.wind[2];  // relative to the medium (exact without wind)
        m3mulTv(lv, Ri, cv);
        m3mulTv(lv + 3, Ri, lin);
        if (m.viscosity > 0) {
          R diam = (box[0] + box[1] + box[2]) / R(3);
          R kr = -R(3.14159265358979323846) * diam * diam * diam * m.viscosity, kl = -R(3) * R(3.14159265358979323846) * diam * m.viscosity;
#pragma unroll
          for (int k = 0; k < 3; k++) { lf[k] = kr * lv[k]; lf[3 + k] = kl * lv[3 + k]; }
        }
        if (m.density > 0) {
          R rho = m.density;
          R b0 = box[0], b1 = box[1], b2 = box[2];
          R b04 = b0 * b0 * b0 * b0, b14 = b1 * b1 * b1 * b1, b24 = b2 * b2 * b2 * b2;
          lf[3] -= R(0.5) * rho * b1 * b2 * r_abs(lv[3]) * lv[3];
          lf[4] -= R(0.5) * rho * b0 * b2 * r_abs(lv[4]) * lv[4];
          lf[5] -= R(0.5) * rho * b0 * b1 * r_abs(lv[5]) * lv[5];
          lf[0] -= rho * b0 * (b14 + b24) * r_abs(lv[0]) * lv[0] / R(64);
          lf[1] -= rho * b1 * (b04 + b24) * r_abs(lv[1]) * lv[1] / R(64);
          lf[2] -= rho * b2 * (b04 + b14) * r_abs(lv[2]) * lv[2] / R(64);
        }
        R tq[3], fr[3], cx[3];
        m3mulv(tq, Ri, lf);
        m3mulv(fr, Ri, lf + 3);
        v3cross(cx, c, fr);
        ff[0] = tq[0] + cx[0]; ff[1] = tq[1] + cx[1]; ff[2] = tq[2] + cx[2];
        ff[3] = fr[0]; ff[4] = fr[1]; ff[5] = fr[2];
      }
#pragma unroll
      for (int e = 0; e < 6; e++) ffl[6 * b + e] = ff[e];
    }
    __syncwarp();
    // per dof: project the subtree sums on the motion axis
    R* bias = p(L.bias); R* passive = p(L.passive);
    const R* damping = dof_damping_of(m, state(), env);
    for (int i = lane; i < m.nv; i += 32) {
      int b0 = m.dof_bodyid[i], b1 = m.body_subtree_end[b0];
      R f[6] = {0, 0, 0, 0, 0, 0}, g[6] = {0, 0, 0, 0, 0, 0};
      for (int b = b0; b < b1; b++) {
#pragma unroll
        for (int e = 0; e < 6; e++) { f[e] += frne[6 * b + e]; g[e] += ffl[6 * b + e]; }
      }
      bias[i] = dot6(cdof + 6 * i, f);
      passive[i] = -damping[i] * qvel[i] + dot6(cdof + 6 * i, g);
    }
    __syncwarp();
    // joint springs: one uniform count test for a model without them
    if (m.nspr > 0) {
      const R* qpos = p(L.qpos);
      for (int k = lane; k < m.nspr; k += 32) {
        int j = m.spr_jnt[k], qa = m.jnt_qposadr[j];
        passive[m.jnt_dofadr[j]] -= m.jnt_stiffness[j] * (qpos[qa] - m.qpos_spring[qa]);
      }
      __syncwarp();
    }
  }

  // ------------------------------------------------------------------------------------------- CRB -> dense M
  DEVN void crb() {
    const DModel<R>& m = model(); const WSLayout& L = lay();
    R* cinert = p(L.cinert);
    const R* armature = dof_armature_of(m, state(), env);
    // composite inertia = sum over the (contiguous, DFS-ordered) subtree, written to scratch
    int nb = m.nbody;
    R* crbuf = p(L.scratch);  // 10 * nbody reals of scratch
    for (int b = lane; b < nb; b += 32) {
      int b1 = m.body_subtree_end[b];
      R acc[10];
#pragma unroll
      for (int k = 0; k < 10; k++) acc[k] = 0;
      for (int c = b; c < b1; c++) {
#pragma unroll
        for (int k = 0; k < 10; k++) acc[k] += cinert[10 * c + k];
      }
#pragma unroll
      for (int k = 0; k < 10; k++) crbuf[10 * b + k] = acc[k];
    }
    __syncwarp();
    // f_i = crb[body(i)] * cdof_i  (stored over cdofdot, which is dead after velocity())
    const R* cdof = p(L.cdof);
    R* fi = p(L.cdofdot);
    for (int i = lane; i < m.nv; i += 32) inert_mulv(fi + 6 * i, crbuf + 10 * m.dof_bodyid[i], cdof + 6 * i);
    R* M = p(L.M);
    int nv = m.nv;
    for (int k = lane; k < nv * nv; k += 32) M[k] = 0;
    __syncwarp();
    for (int e = lane; e < m.nment; e += 32) {
      int i = m.ment_i[e], j = m.ment_j[e];
      R v = dot6(cdof + 6 * j, fi + 6 * i);
      if (i == j) v += armature[i];
      M[i * nv + j] = v;
      M[j * nv + i] = v;
    }
    __syncwarp();
  }

  // ------------------------------------------------------------------------------------------- dense Cholesky
  // A (n x n, row-major, lower part used) -> L in place (lower).  Returns 0 on success (warp-uniform).
  DEVN int chol(R* A, int n) {
    int bad = 0;
    for (int j = 0; j < n; j++) {
      // s_i = A[i][j] - sum_k<j L[i][k] L[j][k] for i >= j
      R djj = 0;
      for (int i = j + lane; i < n; i += 32) {
        R s = A[i * n + j];
        for (int k = 0; k < j; k++) s -= A[i * n + k] * A[j * n + k];
        A[i * n + j] = s;
      }
      __syncwarp();
      djj = A[j * n + j];
      if (!(djj > Lim<R>::minval())) { bad = 1; djj = Lim<R>::minval(); }
      R inv = R(1) / r_sqrt(djj);
      __syncwarp();
      for (int i = j + lane; i < n; i += 32) A[i * n + j] *= inv;
      __syncwarp();
    }
    return bad;
  }
  // x <- (L L^T)^-1 x, x in shared memory (n <= 64)
  DEVN void chol_solve(const R* Lm, R* x, int n) {
    for (int k = 0; k < n; k++) {
      R xk = x[k] / Lm[k * n + k];
      __syncwarp();
      if (lane == 0) x[k] = xk;
      for (int j = k + 1 + lane; j < n; j += 32) x[j] -= Lm[j * n + k] * xk;
      __syncwarp();
    }
    for (int k = n - 1; k >= 0; k--) {
      R xk = x[k] / Lm[k * n + k];
      __syncwarp();
      if (lane == 0) x[k] = xk;
      for (int j = lane; j < k; j += 32) x[j] -= Lm[k * n + j] * xk;
      __syncwarp();
    }
  }


  // x <- (A + dscale*diag(dadd))^-1 x ; A symmetric n x n in shared memory (not modified unless n > 32)
  // blockdiag: the caller guarantees that A has no entries between different kinematic trees
  DEV int spd_solve(R* A, int n, const R* dadd, R dscale, R* x, R* work, bool blockdiag = false) {
    if (blockdiag && n <= 32) {
      const DModel<R>& m = model();
      int ts = m.max_treesize;
      if (ts <= 8) return spd_solve_blk<R, 8>(A, n, dadd, dscale, x, lane, m.dof_treebase, m.dof_treesize);
      if (ts <= 9) return spd_solve_blk<R, 9>(A, n, dadd, dscale, x, lane, m.dof_treebase, m.dof_treesize);
      if (ts <= 12) return spd_solve_blk<R, 12>(A, n, dadd, dscale, x, lane, m.dof_treebase, m.dof_treesize);
    }
    if (n <= 16) return spd_solve_reg<R, 16>(A, n, dadd, dscale, x, lane);
    if (n <= 24) return spd_solve_reg<R, 24>(A, n, dadd, dscale, x, lane);
    if (n <= 32) return spd_solve_reg<R, 32>(A, n, dadd, dscale, x, lane);
    for (int k = lane; k < n * n; k += 32) work[k] = A[k];
    __syncwarp();
    if (dadd) for (int i = lane; i < n; i += 32) work[i * n + i] += dscale * dadd[i];
    __syncwarp();
    int bad = chol(work, n);
    chol_solve(work, x, n);
    return bad;
  }

  // ------------------------------------------------------------------------------------------- actuation
  DEVN void actuation(R* act_force_out) {
    const DModel<R>& m = model(); const WSLayout& L = lay();
    R* qact = p(L.qact);
    const R* ctrl = p(L.ctrl); const R* qpos = p(L.qpos); const R* qvel = p(L.qvel);
    for (int i = lane; i < m.nv; i += 32) qact[i] = 0;
    __syncwarp();
    // each actuator drives one distinct dof in the supported models; accumulate serially per lane-owned actuator
    for (int i = lane; i < m.nu; i += 32) {
      R c = ctrl[i];
      if (m.act_ctrllimited[i]) c = r_clamp(c, m.act_ctrlrange[2 * i], m.act_ctrlrange[2 * i + 1]);
      int j = m.act_trnid[i], qa = m.jnt_qposadr[j], da = m.jnt_dofadr[j];
      R gear = m.act_gear[i];
      R f = m.act_gainprm[3 * i] * c;
      if (m.act_biastype[i]) f += m.act_biasprm[3 * i] + m.act_biasprm[3 * i + 1] * qpos[qa] * gear + m.act_biasprm[3 * i + 2] * qvel[da] * gear;
      if (m.act_forcelimited[i]) f = r_clamp(f, m.act_forcerange[2 * i], m.act_forcerange[2 * i + 1]);
      if (act_force_out) act_force_out[i] = f;
      atomicAdd(&qact[da], gear * f);
    }
    __syncwarp();
  }

  // qfrc_smooth, qacc_smooth = M^-1 qfrc_smooth (factor of M left in H)
  DEVN int acceleration() {
    const DModel<R>& m = model(); const WSLayout& L = lay();
    int nv = m.nv;
    R* qs = p(L.qsmooth); R* qa = p(L.qaccs);
    for (int i = lane; i < nv; i += 32) {
      R v = p(L.passive)[i] - p(L.bias)[i] + p(L.qact)[i];
      qs[i] = v;
      qa[i] = v;
    }
    __syncwarp();
    return spd_solve(p(L.M), nv, (const R*)nullptr, R(0), qa, p(L.H), true);
  }

  // ------------------------------------------------------------------------------------------- Euler
  // semi-implicit Euler with implicit joint damping: (M + h D) a = qfrc_smooth + qfrc_constraint
  DEVN int euler(R* time) {
    const DModel<R>& m = model(); const WSLayout& L = lay();
    int nv = m.nv;
    R h = m.timestep;
    if (vec_bad(p(L.qacc), nv)) {  // mj_checkAcc: reset instead of integrating (returns bit 32; the clock restarts like mj_resetData's)
      for (int i = lane; i < m.nq; i += 32) p(L.qpos)[i] = m.qpos0[i];
      for (int i = lane; i < nv; i += 32) { p(L.qvel)[i] = 0; p(L.qacc)[i] = 0; p(L.qacc_ws)[i] = 0; }
      if (time && lane == 0) *time = 0;
      __syncwarp();
      return 32;
    }
    R* a = p(L.grad);  // reuse solver vector as the integration acceleration
    for (int i = lane; i < nv; i += 32) a[i] = p(L.qsmooth)[i] + p(L.qcon)[i];
    __syncwarp();
    int bad = spd_solve(p(L.M), nv, dof_damping_of(m, state(), env), h, a, p(L.H), true);
    R* qvel = p(L.qvel); R* qpos = p(L.qpos);
    for (int i = lane; i < nv; i += 32) qvel[i] += h * a[i];
    __syncwarp();
    for (int j = lane; j < m.njnt; j += 32) {
      int qa = m.jnt_qposadr[j], da = m.jnt_dofadr[j], t = m.jnt_type[j];
      if (t == JNT_FREE) {
        qpos[qa] += h * qvel[da]; qpos[qa + 1] += h * qvel[da + 1]; qpos[qa + 2] += h * qvel[da + 2];
        R w[3] = {qvel[da + 3], qvel[da + 4], qvel[da + 5]};
        R ang = v3normalize(w) * h;
        R dq[4], r[4], q0[4] = {qpos[qa + 3], qpos[qa + 4], qpos[qa + 5], qpos[qa + 6]};
        aa2quat(dq, w, ang);
        qmul(r, q0, dq);
        qnormalize(r);
        qpos[qa + 3] = r[0]; qpos[qa + 4] = r[1]; qpos[qa + 5] = r[2]; qpos[qa + 6] = r[3];
      } else {
        qpos[qa] += h * qvel[da];
      }
    }
    for (int i = lane; i < nv; i += 32) p(L.qacc_ws)[i] = p(L.qacc)[i];
    if (time && lane == 0) *time += h;
    __syncwarp();
    return bad;
  }
};
