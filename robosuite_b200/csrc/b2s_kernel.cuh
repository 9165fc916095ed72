// Kernels: the fused per-warp step kernel (n_substeps x {step1, controller, step2} with state resident in shared
// memory), reset, and small support kernels.  See include/b2s.h for the reference calls each launch replaces.
#pragma once
#include "b2s_ctrl.cuh"

template <typename R> DEV void load_row(R* dst, const R* src, int n, int lane) {
  for (int i = lane; i < n; i += 32) dst[i] = src[i];
}

// Write-back at the end of step_kernel and of the pipeline's / unit queue's tail: state rows, time and the warn bits of the whole warp -> global memory
template <typename R> DEV void store_state(const Eng<R>& e, int env, R time, int warn) {
  const DModel<R>& m = e.model();
  const DState<R>& s = e.state();
  const WSLayout& L = e.lay();
  const int lane = e.lane;
  const size_t E = env;
  for (int i = lane; i < m.nq; i += 32) s.qpos[E * m.nq + i] = e.p(L.qpos)[i];
  for (int i = lane; i < m.nv; i += 32) {
    s.qvel[E * m.nv + i] = e.p(L.qvel)[i];
    s.qacc[E * m.nv + i] = e.p(L.qacc)[i];
    s.qacc_ws[E * m.nv + i] = e.p(L.qacc_ws)[i];
  }
  warn = warp_or_i(warn);  // some flags (a dropped contact's rows) are raised on the lane that owns the item
  if (lane == 0) { s.time[env] = time; s.warn[env] |= warn; }
  __syncwarp();
}


// The contacts of this substep's step1 -> contact_* / ncon, in static-pair order; rows ncon .. maxcon - 1 get geom -1 and zeros.
// Reads only the contact regions of the workspace, which hold the gathered contacts from collide (fused) or gather_contacts (tail)
// until the next substep: the constraint stage and the solve only read them, and no late load overlays them (layout_tail).
// Compiled once per precision and called by every schedule, so all three write the same bits.
template <typename R>
DEVN void export_contacts(const Eng<R> e, int env, int ncon) {
  const DModel<R>& m = e.model();
  const WSLayout& L = e.lay();
  const DState<R>& s = e.state();
  int lane = e.lane;
  size_t E = env;
  const int* cint = e.pi(L.c_int);
  for (int c = lane; c < m.maxcon; c += 32) {
    bool v = c < ncon;
    s.contact_geom[(E * m.maxcon + c) * 2] = v ? cint[5 * c] : -1;
    s.contact_geom[(E * m.maxcon + c) * 2 + 1] = v ? cint[5 * c + 1] : -1;
    s.contact_dim[E * m.maxcon + c] = v ? cint[5 * c + 2] : 0;
    s.contact_dist[E * m.maxcon + c] = v ? e.p(L.c_dist)[c] : R(0);
    for (int q = 0; q < 3; q++) s.contact_pos[(E * m.maxcon + c) * 3 + q] = v ? e.p(L.c_pos)[3 * c + q] : R(0);
    {
      R f9[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
      if (v) { f9[0] = e.p(L.c_frame)[3 * c]; f9[1] = e.p(L.c_frame)[3 * c + 1]; f9[2] = e.p(L.c_frame)[3 * c + 2]; make_frame(f9); }
      for (int q = 0; q < 9; q++) s.contact_frame[(E * m.maxcon + c) * 9 + q] = f9[q];
    }
    for (int q = 0; q < 3; q++) s.contact_friction[(E * m.maxcon + c) * 3 + q] = v ? e.p(L.c_fric)[3 * c + q] : R(0);
  }
  if (lane == 0) s.ncon[env] = ncon;
}

// The step-1 arrays of this substep -> xpos, xquat, xmat, site_xpos, site_xmat, geom_xpos / geom_xmat of the colliding geoms (the
// others are never computed), qM, cdof, qfrc_bias, qfrc_passive.  Reads the workspace regions kinematics, velocity and crb wrote;
// the fused kernel calls it after collide (whose candidate lists live in the scratch region), phase 0 after publishing its row (its
// layout gives every one of these regions its own words; M over frne / ffl is written by crb after their last use).  Compiled once
// per precision and called by every schedule, so all three write the same bits.
template <typename R>
DEVN void export_kinematics(const Eng<R> e, int env) {
  const DModel<R>& m = e.model();
  const WSLayout& L = e.lay();
  const DState<R>& s = e.state();
  int lane = e.lane;
  size_t E = env;
  load_row(s.xpos + E * 3 * m.nbody, e.p(L.xpos), 3 * m.nbody, lane);
  load_row(s.xquat + E * 4 * m.nbody, e.p(L.xquat), 4 * m.nbody, lane);
  load_row(s.xmat + E * 9 * m.nbody, e.p(L.xmat), 9 * m.nbody, lane);
  load_row(s.site_xpos + E * 3 * m.nsite, e.p(L.spos), 3 * m.nsite, lane);
  load_row(s.site_xmat + E * 9 * m.nsite, e.p(L.smat), 9 * m.nsite, lane);
  for (int k = lane; k < m.ncg; k += 32) {
    int g = m.cg_geom[k];
    for (int q = 0; q < 3; q++) s.geom_xpos[(E * m.ngeom + g) * 3 + q] = e.p(L.gpos)[3 * k + q];
    for (int q = 0; q < 9; q++) s.geom_xmat[(E * m.ngeom + g) * 9 + q] = e.p(L.gmat)[9 * k + q];
  }
  load_row(s.qM + E * m.nv * m.nv, e.p(L.M), m.nv * m.nv, lane);
  load_row(s.cdof + E * 6 * m.nv, e.p(L.cdof), 6 * m.nv, lane);
  load_row(s.qfrc_bias + E * m.nv, e.p(L.bias), m.nv, lane);
  load_row(s.qfrc_passive + E * m.nv, e.p(L.passive), m.nv, lane);
}

// The constraint rows of this substep -> efc_type, efc_aref, efc_D, efc_R (zeros from row nefc on), efc_J (the first nefc * nv
// entries), nefc, and contact_efc_address: a contact's first row, -1 for a contact without rows (not penetrating, or dropped by
// the row budget) and for rows ncon .. maxcon - 1.  Reads J, the row headers and values and the contact headers, which
// make_constraint writes and nothing after it rewrites before the next substep (the controller, actuation, acceleration and the
// solve only read them), so it may run anywhere between make_constraint and the late pose load that overlays J (tail_finish).
template <typename R>
DEVN void export_efc(const Eng<R> e, int env, int ncon, int nefc) {
  const DModel<R>& m = e.model();
  const WSLayout& L = e.lay();
  const DState<R>& s = e.state();
  int lane = e.lane;
  size_t E = env;
  B2S_LOOP
  for (int r = lane; r < m.maxefc; r += 32) {
    bool v = r < nefc;
    s.efc_type[E * m.maxefc + r] = v ? (e.pi(L.e_int)[r] & 255) : 0;
    s.efc_aref[E * m.maxefc + r] = v ? e.p(L.e_aref)[r] : R(0);
    s.efc_D[E * m.maxefc + r] = v ? e.p(L.e_D)[r] : R(0);
    s.efc_R[E * m.maxefc + r] = v ? e.p(L.e_R)[r] : R(0);
  }
  B2S_LOOP
  for (int k = lane; k < nefc * m.nv; k += 32) s.efc_J[E * m.maxefc * m.nv + k] = e.p(L.J)[k];
  const int* cint = e.pi(L.c_int);
  B2S_LOOP
  for (int c = lane; c < m.maxcon; c += 32) s.contact_efc_address[E * m.maxcon + c] = c < ncon ? cint[5 * c + 3] : -1;
  if (lane == 0) s.nefc[env] = nefc;
}

// The step-2 arrays of this substep -> the constraint rows (export_efc), qfrc_actuator, qfrc_smooth, qacc_smooth,
// qfrc_constraint, efc_force (zeros from row nefc on) and solver_niter; runs after the solve, before Euler.  actuator_force is
// written by actuation itself, through the pointer its caller passes on the same substep.  Compiled once per precision and called
// by every schedule (the fused kernel and the tail, right after the solve), so all three write the same bits.
template <typename R>
DEVN void export_dynamics(const Eng<R> e, int env, int ncon, int nefc, int niter) {
  const DModel<R>& m = e.model();
  const WSLayout& L = e.lay();
  const DState<R>& s = e.state();
  int lane = e.lane;
  size_t E = env;
  export_efc(e, env, ncon, nefc);
  B2S_LOOP
  for (int i = lane; i < m.nv; i += 32) {
    s.qfrc_actuator[E * m.nv + i] = e.p(L.qact)[i];
    s.qfrc_smooth[E * m.nv + i] = e.p(L.qsmooth)[i];
    s.qacc_smooth[E * m.nv + i] = e.p(L.qaccs)[i];
    s.qfrc_constraint[E * m.nv + i] = e.p(L.qcon)[i];
  }
  B2S_LOOP
  for (int r = lane; r < m.maxefc; r += 32) s.efc_force[E * m.maxefc + r] = r < nefc ? e.p(L.e_force)[r] : R(0);
  if (lane == 0) s.solver_niter[env] = niter;
}

template <typename R>
__global__ void __launch_bounds__(512, 1) step_kernel(int phases, int nsub, const R* action, int slot, const uint8_t* mask = nullptr) {
  const DModel<R>& m = cmodel<R>(slot);
  const DState<R>& s = cstate<R>(slot);
  const WSLayout& L = c_lay[slot][LAY_FULL];
  extern __shared__ __align__(16) unsigned char smem_raw[];
  R* smem = reinterpret_cast<R*>(smem_raw);
  int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  int env = blockIdx.x * wpb + warp;
  // every warp of the block runs the phase sequence (block barriers keep the warps of an SM in the same code
  // region, which is what bounds the instruction-cache working set); warps beyond n_env shadow the last env
  bool live = env < s.n_env;
  if (!live) env = s.n_env - 1;
  if (mask) {
    // masked launch (forward pass of the environments being reset): blocks without a selected environment leave, the other warps of a
    // block shadow a selected one (they write the same values to the same addresses, like the tail warps above)
    __shared__ int pick;
    if (threadIdx.x == 0) pick = -1;
    __syncthreads();
    live = live && mask[env];
    if (live && lane == 0) atomicMax(&pick, env);
    __syncthreads();
    if (pick < 0) return;
    if (!live) env = pick;
  }
  Eng<R> e(smem + (size_t)warp * L.fused_stride, lane, slot, LAY_FULL);
  e.env = env;
  size_t E = env;
  load_row(e.p(L.qpos), s.qpos + E * m.nq, m.nq, lane);
  load_row(e.p(L.qvel), s.qvel + E * m.nv, m.nv, lane);
  load_row(e.p(L.qacc), s.qacc + E * m.nv, m.nv, lane);
  load_row(e.p(L.qacc_ws), s.qacc_ws + E * m.nv, m.nv, lane);
  load_row(e.p(L.ctrl), s.ctrl + E * m.nu, m.nu, lane);
  R time = s.time[env];
  CtrlState<R> cs;
  if (phases & PH_CTRL) ctrl_load(e, cs, env);
  __syncwarp();
  int warn = 0;
  for (int sub = 0; sub < nsub; sub++) {
    int ncon = 0, nefc = 0, niter = 0;
    const bool last = live && sub == nsub - 1, ex = last && (phases & PH_EXPORT);
    const int xm = ex ? EXP_ALL : last ? s.export_con | s.export_kin | s.export_dyn : 0;  // the array groups this substep writes
    __syncthreads();
    if (phases & PH_STEP1) {
      if (e.kinematics()) {  // diverged state reset to the model defaults (mj_checkPos / mj_checkVel)
        for (int i = lane; i < m.nv; i += 32) { e.p(L.qacc)[i] = 0; e.p(L.qacc_ws)[i] = 0; }
        time = 0; warn |= 32;
        __syncwarp();
      }
      e.velocity();
      e.crb();
      __syncthreads();
      ncon = collide(e, warn);
      if (xm & EXP_STEP1) export_kinematics(e, env);
      if (xm & EXP_CONTACTS) export_contacts(e, env, ncon);
      __syncthreads();
      nefc = make_constraint(e, ncon, warn);
      if (ex && !(phases & PH_STEP2)) export_efc(e, env, ncon, nefc);  // b2s_step1: no solve follows, the rows alone
    }
    // a shadow warp skips the controller: the joint controllers update their state in HBM in place, and a second warp doing so
    // for the same environment would race it (the joint-velocity integral and derivative ring taking the substep twice)
    if (live && (phases & PH_CTRL)) ctrl_run(e, cs, env, sub == 0 ? action : (const R*)nullptr);
    if (phases & PH_STEP2) {
      const bool dyn = (xm & EXP_STEP2) != 0;
      e.actuation(dyn ? s.actuator_force + E * m.nu : nullptr);
      if (e.acceleration()) warn |= 1;
      __syncthreads();
      niter = solve(e, nefc, ncon, warn);
      if (dyn) export_dynamics(e, env, ncon, nefc, niter);
      if (!(phases & PH_NOINTEGRATE)) {
        { int eb = e.euler(&time); if (eb & 32) warn |= 32; else if (eb) warn |= 2; }
      }
    }
    if (live && (phases & PH_OBS) && c_cc[slot].obs_dim > 0) {
      // The reference's observables sample on the LAST substep of a control step at the default rate: reset()'s forced update
      // already advances their period timer by one model timestep (utils/observables.py:214-259, environments/base.py:418-427),
      // so the period closes after substep 24 and the next update - substep 25 - takes the sample.  Other rates: obs_due.
      const bool last = sub == nsub - 1, only_fresh = (phases & PH_NOINTEGRATE) != 0;
      const unsigned due = obs_due(e, env, last, only_fresh);
      if (due) write_obs(e, env, only_fresh, due);
      if (last) write_task(e, env, ncon);
    }
    __syncwarp();
  }
  if (!live) return;
  if (phases & PH_CTRL) {
    for (int i = lane; i < m.nu; i += 32) s.ctrl[E * m.nu + i] = e.p(L.ctrl)[i];
    ctrl_store(e, cs, env);
  }
  store_state(e, env, time, warn);
}

// masked episode reset without a host round trip: selected environments take their generalized positions from `qpos_new` (a pool of
// sampled initial states, [n_env, nq]; nullptr: the model's qpos0), everything else is cleared the way reset_kernel does.  `carry`
// (nullptr without a placement program): warn bits b2s_place_objects left for this reset, which it takes and clears
template <typename R>
__global__ void reset_envs_kernel(const uint8_t* mask, const R* qpos_new, int slot, int* carry) {
  const DModel<R>& m = cmodel<R>(slot);
  const DState<R>& s = cstate<R>(slot);
  int env = blockIdx.x * blockDim.x + threadIdx.x;
  if (env >= s.n_env) return;
  if (mask && !mask[env]) return;
  size_t E = env;
  for (int i = 0; i < m.nq; i++) s.qpos[E * m.nq + i] = qpos_new ? qpos_new[E * m.nq + i] : m.qpos0[i];
  for (int i = 0; i < m.nv; i++) { s.qvel[E * m.nv + i] = 0; s.qacc[E * m.nv + i] = 0; s.qacc_ws[E * m.nv + i] = 0; }
  for (int i = 0; i < m.nu; i++) s.ctrl[E * m.nu + i] = 0;
  s.time[env] = 0;
  s.warn[env] = carry ? carry[env] : 0;
  if (carry) carry[env] = 0;
  if (s.obs_fresh) s.obs_fresh[env] = 1;
}

// ---- set-constants pass (b2s_set_const): the compiler's _set_const (mjcf/compiler.py) for the masked environments, one warp each,
// from the environment's own masses, moments and sizes.  Kinematics and CRB at qpos0 (world-pose overrides honoured) give M, then
//   meaninertia       = mean diag(M)
//   dof_invweight0    = diag(M^-1), averaged over the translational and the rotational block of each free joint
//   body_invweight0   = (mean translational, mean rotational) diagonal of J M^-1 J^T, J = Jacobian of the body's centre of mass
// and every overridden geom gets its bounding radius and local box from its size (the compiler's per-type rules).  The CRB adds the
// environment's own armature.  Override values that are non-finite or non-positive (damping, armature and friction loss: negative),
// a non-finite solref / solimp component, or moments that violate the triangle inequality set warn bit 128.
// Workspace per warp: the fused layout followed by nv * nv words for M^-1 (`stride` words in all).
template <typename R>
__global__ void __launch_bounds__(512, 1) set_const_kernel(const uint8_t* mask, int slot, int stride) {
  const DModel<R>& m = cmodel<R>(slot);
  const DState<R>& s = cstate<R>(slot);
  const WSLayout& L = c_lay[slot][LAY_FULL];
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  const int env = blockIdx.x * wpb + warp;
  if (env >= s.n_env || (mask && !mask[env])) return;
  Eng<R> e(reinterpret_cast<R*>(smem_raw) + (size_t)warp * stride, lane, slot, LAY_FULL);
  e.env = env;
  const int nv = m.nv, nb = m.nbody;
  const size_t E = env;
  auto pos = [](R v) { return isfinite(v) && v > R(0); };
  int bad = 0;
  for (int k = lane; k < s.n_mg; k += 32) {
    const size_t o = (size_t)k * s.n_env + E;
    const int t = m.geom_type[s.mg_id[k]];
    const R* sz = s.mg_size + 3 * o;
    const R* fr = s.mg_fric + 3 * o;
    const int nsz = t == G_SPHERE ? 1 : (t == G_CAPSULE || t == G_CYLINDER ? 2 : 3);
    for (int q = 0; q < 3; q++) if (!pos(fr[q]) || (q < nsz && !pos(sz[q]))) bad = 1;
    for (int q = 0; q < 2; q++) if (!isfinite(s.mg_solref[2 * o + q])) bad = 1;
    for (int q = 0; q < 5; q++) if (!isfinite(s.mg_solimp[5 * o + q])) bad = 1;
    R r = sz[0], h = sz[1], rb, hx = r, hy = r, hz = r;
    if (t == G_SPHERE) rb = r;
    else if (t == G_CAPSULE) { rb = r + h; hz = r + h; }
    else if (t == G_CYLINDER) { rb = r_sqrt(r * r + h * h); hz = h; }
    else {  // ellipsoid, box
      hx = sz[0]; hy = sz[1]; hz = sz[2];
      rb = t == G_ELLIPSOID ? r_max(r_max(hx, hy), hz) : r_sqrt(hx * hx + hy * hy + hz * hz);
    }
    s.mg_rbound[o] = rb;
    R* a = s.mg_aabb + 6 * o;
    a[0] = 0; a[1] = 0; a[2] = 0; a[3] = hx; a[4] = hy; a[5] = hz;
  }
  for (int k = lane; k < s.n_mb; k += 32) {
    const size_t o = (size_t)k * s.n_env + E;
    const R* I = s.mb_inertia + 3 * o;
    if (!pos(s.mb_mass[o]) || !pos(I[0]) || !pos(I[1]) || !pos(I[2]) || I[0] + I[1] < I[2] || I[0] + I[2] < I[1] || I[1] + I[2] < I[0]) bad = 1;
  }
  auto nonneg = [](R v) { return isfinite(v) && v >= R(0); };
  const R* dofv[3] = {s.dof_damp, s.dof_arm, s.dof_floss};
  for (int k = 0; k < 3; k++)
    if (dofv[k]) for (int i = lane; i < nv; i += 32) if (!nonneg(dofv[k][E * nv + i])) bad = 1;
  bad = warp_or_i(bad);
  if (bad && lane == 0) s.warn[env] |= 128;
  // M at qpos0
  for (int i = lane; i < m.nq; i += 32) e.p(L.qpos)[i] = m.qpos0[i];
  for (int i = lane; i < nv; i += 32) e.p(L.qvel)[i] = 0;
  __syncwarp();
  e.kinematics();
  e.crb();
  const R* M = e.p(L.M);
  R tr = 0;
  for (int i = 0; i < nv; i++) tr += M[i * nv + i];
  if (lane == 0) s.mean_inertia[env] = nv > 0 ? tr / R(nv) : R(1);
  // M^-1, column by column from one Cholesky factor (in H)
  R* H = e.p(L.H); R* x = e.p(L.grad); R* Mi = e.ws + L.total;
  for (int k = lane; k < nv * nv; k += 32) H[k] = M[k];
  __syncwarp();
  e.chol(H, nv);
  for (int c = 0; c < nv; c++) {
    for (int i = lane; i < nv; i += 32) x[i] = i == c ? R(1) : R(0);
    __syncwarp();
    e.chol_solve(H, x, nv);
    for (int i = lane; i < nv; i += 32) Mi[i * nv + c] = x[i];
    __syncwarp();
  }
  for (int i = lane; i < nv; i += 32) {
    int j = m.dof_jntid[i], b = i;
    R v = Mi[i * nv + i];
    if (m.jnt_type[j] == JNT_FREE) {
      b = m.jnt_dofadr[j] + (i - m.jnt_dofadr[j] < 3 ? 0 : 3);
      v = (Mi[b * nv + b] + Mi[(b + 1) * nv + b + 1] + Mi[(b + 2) * nv + b + 2]) / R(3);
    }
    s.dof_iw[E * nv + i] = v;
  }
  const R* cdof = e.p(L.cdof); const R* xipos = e.p(L.xipos);
  for (int b = lane; b < nb; b += 32) {
    R at = 0, ar = 0;
    if (b > 0 && m.body_weldid[b] != 0) {
      const R* p = xipos + 3 * b;
      const unsigned long long chain = m.body_dofmask[b];
      for (int i = 0; i < nv; i++) {
        if (!((chain >> i) & 1ull)) continue;
        const R* ci = cdof + 6 * i;
        R pi[3];
        v3cross(pi, ci, p);
        pi[0] += ci[3]; pi[1] += ci[4]; pi[2] += ci[5];
        for (int j = 0; j < nv; j++) {
          if (!((chain >> j) & 1ull)) continue;
          const R* cj = cdof + 6 * j;
          R pj[3];
          v3cross(pj, cj, p);
          pj[0] += cj[3]; pj[1] += cj[4]; pj[2] += cj[5];
          const R w = Mi[i * nv + j];
          at += w * v3dot(pi, pj);
          ar += w * v3dot(ci, cj);
        }
      }
    }
    s.body_iw[(E * nb + b) * 2] = at / R(3);
    s.body_iw[(E * nb + b) * 2 + 1] = ar / R(3);
  }
}

// ---- device perturbation of the override arrays (b2s_perturb_model), the batched counterpart of the reference's DynamicsModder
// (utils/mjmod.py): every configured (field, id) of the masked environments is redrawn around the MODEL's value.
//   scale: v = v_model * (1 + d)       shift: v = max(0, v_model + d)       d = a * (2u - 1), u in [0, 1)
// u comes from Philox4x32-10 (Salmon et al., SC'11) keyed by the seed, counter (env, call counter, entry, component), so an
// environment's draws do not depend on n_env or on the mask.  u = 53 bits of the first two output words.  The arithmetic is in fp64
// with explicit roundings (no contraction), so a host restatement reproduces every bit; the result is rounded to the handle's precision.
struct PerturbEntry { void* dst; int stride, mode, one_draw; double amp; };  // value of (env, component c) at dst[env * stride + c]
struct PerturbItem { int entry, comp; double model; };                     // one per (entry, component), in entry order

template <typename R>
__global__ void perturb_kernel(const PerturbEntry* ent, const PerturbItem* item, int nitems, int n_env, const uint8_t* mask,
                               unsigned long long seed, unsigned counter) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)n_env * nitems) return;
  const int env = (int)(t / nitems), it = (int)(t % nitems);
  if (mask && !mask[env]) return;
  const PerturbItem p = item[it];
  const PerturbEntry& en = ent[p.entry];
  const uint4 x = philox4x32_10(make_uint4((unsigned)env, counter, (unsigned)p.entry, en.one_draw ? 0u : (unsigned)p.comp),
                                (unsigned)seed, (unsigned)(seed >> 32));
  const double u = (double)(((unsigned long long)(x.x >> 5) << 26) | (x.y >> 6)) * 0x1p-53;
  const double d = __dmul_rn(en.amp, __dsub_rn(__dmul_rn(2.0, u), 1.0));
  const double v = en.mode == 0 ? __dmul_rn(p.model, __dadd_rn(1.0, d)) : fmax(0.0, __dadd_rn(p.model, d));
  reinterpret_cast<R*>(en.dst)[(size_t)env * en.stride + p.comp] = (R)v;
}

template <typename R>
__global__ void reset_kernel(const uint8_t* mask, int slot) {
  const DModel<R>& m = cmodel<R>(slot);
  const DState<R>& s = cstate<R>(slot);
  int env = blockIdx.x * blockDim.x + threadIdx.x;
  if (env >= s.n_env) return;
  if (mask && !mask[env]) return;
  size_t E = env;
  for (int i = 0; i < m.nq; i++) s.qpos[E * m.nq + i] = m.qpos0[i];
  for (int i = 0; i < m.nv; i++) { s.qvel[E * m.nv + i] = 0; s.qacc[E * m.nv + i] = 0; s.qacc_ws[E * m.nv + i] = 0; }
  for (int i = 0; i < m.nu; i++) s.ctrl[E * m.nu + i] = 0;
  s.time[env] = 0;
  s.warn[env] = 0;
}

// per-episode hidden state of the collision pipeline: the GJK warm-start directions of the environments being reset
// (a replay from a restored state must not depend on what ran before: tests/test_environments/test_action_playback.py)
template <typename R>
__global__ void cache_reset_kernel(const uint8_t* mask, int slot) {
  const DModel<R>& m = cmodel<R>(slot);
  const DState<R>& s = cstate<R>(slot);
  if (!s.gjk_cache) return;
  size_t per = (size_t)m.npair * 3, idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= per * (size_t)s.n_env) return;
  if (mask && !mask[idx / per]) return;
  s.gjk_cache[idx] = 0;
}

// flattened simulator state [time, qpos, qvel] per environment <-> the state arrays (MjSimState.flatten, binding_utils.py:56-70)
template <typename R>
__global__ void state_io_kernel(R* flat, int set, int slot) {
  const DModel<R>& m = cmodel<R>(slot);
  const DState<R>& s = cstate<R>(slot);
  const int w = 1 + m.nq + m.nv;
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (size_t)s.n_env * w) return;
  size_t env = idx / w; int k = (int)(idx % w);
  R* p = k == 0 ? s.time + env : (k <= m.nq ? s.qpos + env * m.nq + (k - 1) : s.qvel + env * m.nv + (k - 1 - m.nq));
  if (set) *p = flat[idx]; else flat[idx] = *p;
}

// Jacobian of a point that moves with `body` (body frame origin: kind 0, geom centre: kind 1, site: the dedicated kernel below)
template <typename R>
__global__ void jac_point_kernel(int kind, int id, R* jacp, R* jacr, int slot) {
  const DModel<R>& m = cmodel<R>(slot);
  const DState<R>& s = cstate<R>(slot);
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= s.n_env * m.nv) return;
  int env = idx / m.nv, i = idx % m.nv;
  size_t E = env;
  int body = kind == 0 ? id : m.geom_bodyid[id];
  const R* pos = kind == 0 ? s.xpos + (E * m.nbody + id) * 3 : s.geom_xpos + (E * m.ngeom + id) * 3;
  bool on = (m.body_dofmask[body] >> i) & 1ull;
  const R* cd = s.cdof + (E * m.nv + i) * 6;
  R t[3] = {0, 0, 0}, w[3] = {0, 0, 0};
  if (on) {
    v3cross(t, cd, pos);
    t[0] += cd[3]; t[1] += cd[4]; t[2] += cd[5];
    w[0] = cd[0]; w[1] = cd[1]; w[2] = cd[2];
  }
  for (int r = 0; r < 3; r++) {
    if (jacp) jacp[(E * 3 + r) * m.nv + i] = t[r];
    if (jacr) jacr[(E * 3 + r) * m.nv + i] = w[r];
  }
}

// translational / rotational Jacobian of a site from the exported cdof and site_xpos (valid after forward/step1)
template <typename R>
__global__ void jac_site_kernel(int site, R* jacp, R* jacr, int slot) {
  const DModel<R>& m = cmodel<R>(slot);
  const DState<R>& s = cstate<R>(slot);
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= s.n_env * m.nv) return;
  int env = idx / m.nv, i = idx % m.nv;
  size_t E = env;
  int body = m.site_bodyid[site];
  bool on = (m.body_dofmask[body] >> i) & 1ull;
  const R* cd = s.cdof + (E * m.nv + i) * 6;
  const R* pos = s.site_xpos + (E * m.nsite + site) * 3;
  R t[3] = {0, 0, 0}, w[3] = {0, 0, 0};
  if (on) {
    v3cross(t, cd, pos);
    t[0] += cd[3]; t[1] += cd[4]; t[2] += cd[5];
    w[0] = cd[0]; w[1] = cd[1]; w[2] = cd[2];
  }
  for (int r = 0; r < 3; r++) {
    if (jacp) jacp[(E * 3 + r) * m.nv + i] = t[r];
    if (jacr) jacr[(E * 3 + r) * m.nv + i] = w[r];
  }
}
