// Per-warp soft-constraint assembly (friction-loss dofs, joint limits, elliptic-cone contacts) and primal Newton
// solver with exact line search; rows / contacts / Hessian entries are split across lanes.
// Replaces the constraint stage of mj_step1 and the solve of mj_step2 (robosuite/utils/binding_utils.py:1101-1107),
// SURVEY.md section 8 rows a1/a7 and Appendix C.
#pragma once
// B2S_LOOP: the loops of make_constraint / constraint_update / ls_eval / solve keep their rolled form.  Unrolled, `solve` alone
// is 90 KB of SASS against a 32 KB instruction cache; rolled it is 31 KB and the whole step is 11.7 % faster (239 k -> 267 k
// env-steps/s, Lift 4096 envs).
#define B2S_LOOP _Pragma("unroll 1")
#include "b2s_collide.cuh"

#define B2S_MINIMP 0.0001
#define B2S_MAXIMP 0.9999

template <typename R> DEV R impedance(const R* solimp, R pos, R margin) {
  R dmin = r_clamp(solimp[0], R(B2S_MINIMP), R(B2S_MAXIMP)), dmax = r_clamp(solimp[1], R(B2S_MINIMP), R(B2S_MAXIMP));
  R width = r_max(R(0), solimp[2]), mid = r_clamp(solimp[3], R(B2S_MINIMP), R(B2S_MAXIMP)), power = r_max(R(1), solimp[4]);
  if (dmin == dmax || width <= Lim<R>::minval()) return R(0.5) * (dmin + dmax);
  R x = r_abs(pos - margin) / width;
  if (x >= 1) return dmax;
  if (x <= 0) return dmin;
  R y;
  if (power == 1) y = x;
  else if (power == 2) y = x <= mid ? x * x / mid : 1 - (1 - x) * (1 - x) / (1 - mid);
  else if (x <= mid) y = r_pow(x, power) / r_pow(mid, power - 1);
  else y = 1 - r_pow(1 - x, power) / r_pow(1 - mid, power - 1);
  return dmin + y * (dmax - dmin);
}

template <typename R> DEV void kb_from_solref(const R* solref, R dmax, R timestep, R& K, R& B) {
  if (solref[0] > 0) {
    R tc = r_max(solref[0], 2 * timestep), dr = solref[1];
    K = R(1) / r_max(Lim<R>::minval(), dmax * dmax * tc * tc * dr * dr);
    B = R(2) / r_max(Lim<R>::minval(), dmax * tc);
  } else {
    K = -solref[0] / r_max(Lim<R>::minval(), dmax * dmax);
    B = -solref[1] / r_max(Lim<R>::minval(), dmax);
  }
}

// friction coefficient of contact row k >= 1 (rows 1,2 sliding; 3 torsional; 4,5 rolling)
template <typename R> DEV R row_friction(const R* f3, int k) { return k <= 2 ? f3[0] : (k == 3 ? f3[1] : f3[2]); }

// Builds all constraint rows in the workspace.  Returns nefc (warp-uniform).
template <typename R> DEVN int make_constraint(Eng<R> e, int ncon, int& warn) {
  const DModel<R>& m = e.model();
  const WSLayout& L = e.lay();
  int lane = e.lane, nv = m.nv;
  R* J = e.p(L.J);
  R* eD = e.p(L.e_D); R* eR = e.p(L.e_R); R* earef = e.p(L.e_aref); R* efl = e.p(L.e_floss);
  R* epos = e.p(L.e_jar);  // efc_pos is only needed while building rows: borrow jar
  int* eint = e.pi(L.e_int);
  const R* qpos = e.p(L.qpos); const R* qvel = e.p(L.qvel);
  int nefc = 0;
  const DState<R>& st = e.state();
  if (!st.dof_floss) {
    // --- friction-loss rows (static list)
    B2S_LOOP
    for (int r = lane; r < m.nfl; r += 32) {
      int dof = m.fl_dof[r];
      B2S_LOOP
      for (int i = 0; i < nv; i++) J[r * nv + i] = i == dof ? R(1) : R(0);
      eint[r] = C_FRICTION | (dof << 8);
      epos[r] = 0;
      efl[r] = m.dof_frictionloss[dof];
    }
    nefc = m.nfl;
  } else {
    // --- friction-loss rows of this environment (b2s_model_override "dof_frictionloss"): its dofs with a value > 0, in dof order
    const R* floss = st.dof_floss + (size_t)e.env * nv;
    B2S_LOOP
    for (int base = 0; base < nv; base += 32) {
      int dof = base + lane;
      R fl = dof < nv ? floss[dof] : R(0);
      int act = fl > 0;
      unsigned mask = __ballot_sync(B2S_FULL, act);
      int r = nefc + __popc(mask & ((1u << lane) - 1));
      if (act && r < L.me) {
        B2S_LOOP
        for (int i = 0; i < nv; i++) J[r * nv + i] = i == dof ? R(1) : R(0);
        eint[r] = C_FRICTION | (dof << 8);
        epos[r] = 0;
        efl[r] = fl;
      }
      nefc += __popc(mask);
    }
  }
  // --- joint limits: candidate k is side k & 1 (lower first) of limited joint k >> 1.  A side is active within its joint's margin,
  // so a range narrower than twice the margin has both rows.  The row's pos is dist - margin: impedance and aref take it as is.
  B2S_LOOP
  for (int base = 0; base < 2 * m.nlim; base += 32) {
    int k = base + lane, act = 0, j = 0, upper = 0;
    R dist = 0;
    if (k < 2 * m.nlim) {
      j = m.lim_jnt[k >> 1];
      upper = k & 1;
      R value = qpos[m.jnt_qposadr[j]], margin = m.jnt_margin[j];
      dist = upper ? m.jnt_range[2 * j + 1] - value : value - m.jnt_range[2 * j];
      act = dist < margin;
      dist -= margin;
    }
    unsigned mask = __ballot_sync(B2S_FULL, act);
    if (act) {
      int r = nefc + __popc(mask & ((1u << lane) - 1));
      if (r < L.me) {
        int dof = m.jnt_dofadr[j];
        B2S_LOOP
        for (int i = 0; i < nv; i++) J[r * nv + i] = i == dof ? R(upper ? -1 : 1) : R(0);
        eint[r] = C_LIMIT | (j << 8);
        epos[r] = dist;
        efl[r] = 0;
      }
    }
    nefc += __popc(mask);
  }
  if (nefc > L.me) { nefc = L.me; warn |= 8; }
  // --- contacts: row addresses by ordered prefix sum over active contacts
  int* cint = e.pi(L.c_int);
  const R* cdist = e.p(L.c_dist);
  int first_contact_row = nefc;
  B2S_LOOP
  for (int base = 0; base < ncon; base += 32) {
    int c = base + lane, dim = 0;
    if (c < ncon && cdist[c] < 0) dim = cint[5 * c + 2];
    int off = dim;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(B2S_FULL, off, o); if (lane >= o) off += t; }
    int total = __shfl_sync(B2S_FULL, off, 31);
    int adr = nefc + off - dim;
    if (c < ncon) {
      if (dim > 0 && adr + dim <= L.me) cint[5 * c + 3] = adr;
      else { cint[5 * c + 3] = -1; if (dim > 0) warn |= 8; }
    }
    nefc += total;
  }
  if (nefc > L.me) nefc = L.me;  // rows of dropped contacts are simply absent (flagged in warn)
  __syncwarp();
  // recompute exact nefc as end of the last placed contact
  {
    int last = first_contact_row;
    B2S_LOOP
    for (int c = lane; c < ncon; c += 32)
      if (cint[5 * c + 3] >= 0) last = max(last, cint[5 * c + 3] + cint[5 * c + 2]);
    B2S_LOOP
    for (int o = 16; o > 0; o >>= 1) last = max(last, __shfl_xor_sync(B2S_FULL, last, o));
    nefc = last;
  }
  // row headers of contact rows
  B2S_LOOP
  for (int c = lane; c < ncon; c += 32) {
    int adr = cint[5 * c + 3];
    if (adr < 0) continue;
    int dim = cint[5 * c + 2];
    B2S_LOOP
    for (int k = 0; k < dim; k++) {
      eint[adr + k] = (dim == 1 ? C_FRICTIONLESS : C_ELLIPTIC) | (c << 8);
      epos[adr + k] = k == 0 ? cdist[c] : R(0);
      efl[adr + k] = 0;
    }
  }
  __syncwarp();
  // full contact frames (normal, two tangents) into scratch
  {
    R* fr = e.p(L.scratch);
    const R* cn = e.p(L.c_frame);
    B2S_LOOP
    for (int c = lane; c < ncon; c += 32) {
      R f9[9] = {cn[3 * c], cn[3 * c + 1], cn[3 * c + 2], 0, 0, 0, 0, 0, 0};
      make_frame(f9);
#pragma unroll
      for (int q = 0; q < 9; q++) fr[9 * c + q] = f9[q];
    }
  }
  __syncwarp();
  // contact Jacobian: work items = (row, dof)
  {
    const R* cdof = e.p(L.cdof); const R* cpos = e.p(L.c_pos); const R* cfr = e.p(L.scratch);
    int nrows = nefc - first_contact_row;
    B2S_LOOP
    for (int w = lane; w < nrows * nv; w += 32) {
      int r = first_contact_row + w / nv, i = w % nv;
      int c = eint[r] >> 8, k = r - cint[5 * c + 3];
      int b1 = m.geom_bodyid[cint[5 * c]], b2 = m.geom_bodyid[cint[5 * c + 1]];
      int s = (int)((m.body_dofmask[b2] >> i) & 1ull) - (int)((m.body_dofmask[b1] >> i) & 1ull);
      R v = 0;
      if (s != 0) {
        const R* cd = cdof + 6 * i;
        const R* ax = cfr + 9 * c + 3 * (k < 3 ? k : k - 3);
        if (k < 3) {
          R t[3];
          v3cross(t, cd, cpos + 3 * c);
          v = ax[0] * (cd[3] + t[0]) + ax[1] * (cd[4] + t[1]) + ax[2] * (cd[5] + t[2]);
        } else v = ax[0] * cd[0] + ax[1] * cd[1] + ax[2] * cd[2];
        v *= R(s);
      }
      J[r * nv + i] = v;
    }
  }
  __syncwarp();
  // per row: velocity, impedance, regularisation, reference acceleration
  R* ejv = e.p(L.e_jv);  // borrow: holds imp of each row until the cone pass
  B2S_LOOP
  for (int r = lane; r < nefc; r += 32) {
    R vel = 0;
    B2S_LOOP
    for (int i = 0; i < nv; i++) vel += J[r * nv + i] * qvel[i];
    int type = eint[r] & 255, id = eint[r] >> 8;
    R solref[2], solimp[5], diag;
    int first = 1;
    if (type == C_FRICTION) {
      solref[0] = m.dof_solref[2 * id]; solref[1] = m.dof_solref[2 * id + 1];
      B2S_LOOP
      for (int q = 0; q < 5; q++) solimp[q] = m.dof_solimp[5 * id + q];
      diag = dof_invweight0_of(m, e.state(), e.env)[id];
    } else if (type == C_LIMIT) {
      solref[0] = m.jnt_solref[2 * id]; solref[1] = m.jnt_solref[2 * id + 1];
      B2S_LOOP
      for (int q = 0; q < 5; q++) solimp[q] = m.jnt_solimp[5 * id + q];
      diag = dof_invweight0_of(m, e.state(), e.env)[m.jnt_dofadr[id]];
    } else {
      int g1 = cint[5 * id], g2 = cint[5 * id + 1], k = r - cint[5 * id + 3];
      first = k == 0;
      int b1 = m.geom_bodyid[g1], b2 = m.geom_bodyid[g2];
      const R* biw = body_invweight0_of(m, e.state(), e.env);
      const R* sr1 = geom_solref_of(m, e.state(), g1, e.env); const R* sr2 = geom_solref_of(m, e.state(), g2, e.env);
      const R* si1 = geom_solimp_of(m, e.state(), g1, e.env); const R* si2 = geom_solimp_of(m, e.state(), g2, e.env);
      diag = k < 3 ? biw[2 * b1] + biw[2 * b2] : biw[2 * b1 + 1] + biw[2 * b2 + 1];
      // solref / solimp mixing (solmix-weighted)
      R s1 = m.geom_solmix[g1], s2 = m.geom_solmix[g2], mix;
      int p1 = m.geom_priority[g1], p2 = m.geom_priority[g2];
      if (p1 != p2) mix = p1 > p2 ? R(1) : R(0);
      else if (s1 >= Lim<R>::minval() && s2 >= Lim<R>::minval()) mix = s1 / (s1 + s2);
      else if (s1 < Lim<R>::minval() && s2 < Lim<R>::minval()) mix = R(0.5);
      else mix = s1 < Lim<R>::minval() ? R(0) : R(1);
      R r10 = sr1[0], r11 = sr1[1], r20 = sr2[0], r21 = sr2[1];
      if (p1 != p2 || (r10 > 0 && r20 > 0)) { solref[0] = mix * r10 + (1 - mix) * r20; solref[1] = mix * r11 + (1 - mix) * r21; }
      else { solref[0] = r_min(r10, r20); solref[1] = r_min(r11, r21); }
      B2S_LOOP
      for (int q = 0; q < 5; q++) solimp[q] = mix * si1[q] + (1 - mix) * si2[q];
    }
    R pos = epos[r];
    // friction rows of a cone reuse the normal row's impedance: evaluate it from the normal's pos
    R posn = first ? pos : e.p(L.c_dist)[id];
    R imp = impedance(solimp, posn, R(0));
    R dmax = r_clamp(solimp[1], R(B2S_MINIMP), R(B2S_MAXIMP));
    R K, B;
    kb_from_solref(solref, dmax, m.timestep, K, B);
    if (type == C_FRICTION || (type == C_ELLIPTIC && !first)) K = 0;
    eR[r] = r_max(Lim<R>::minval(), (1 - imp) * diag / imp);
    earef[r] = -B * vel - K * imp * pos;
    ejv[r] = imp;
  }
  __syncwarp();
  // elliptic cones: friction-row regularisation and cone coefficient mu
  const R* cfric = e.p(L.c_fric);
  B2S_LOOP
  for (int c = lane; c < ncon; c += 32) {
    int adr = cint[5 * c + 3], dim = cint[5 * c + 2];
    if (adr < 0 || dim < 3) continue;
    R f0 = cfric[3 * c];
    R R0 = eR[adr];
    R R1 = R0 / r_max(Lim<R>::minval(), m.impratio);
    eR[adr + 1] = R1;
    B2S_LOOP
    for (int k = 2; k < dim; k++) { R fk = row_friction(cfric + 3 * c, k); eR[adr + k] = R1 * f0 * f0 / (fk * fk); }
    efl[adr] = f0 * r_sqrt(R1 / R0);  // cone coefficient mu, kept in the (otherwise unused) frictionloss slot
  }
  __syncwarp();
  B2S_LOOP
  for (int r = lane; r < nefc; r += 32) eD[r] = R(1) / eR[r];
  __syncwarp();
  return nefc;
}

// ---------------------------------------------------------------------------------------------- solver pieces
// Evaluate all constraints at jar (in workspace): forces, per-row active curvature (e_jv borrowed as `act`), cone
// Hessian blocks (scratch), returns total constraint cost (warp-uniform).  If hess==0 only cost/forces.
template <typename R>
DEVN R constraint_update(Eng<R> e, int nefc, int ncon, bool hess) {
  const DModel<R>& m = e.model();
  const WSLayout& L = e.lay();
  int lane = e.lane;
  const R* jar = e.p(L.e_jar); const R* eD = e.p(L.e_D); const R* eR = e.p(L.e_R); const R* efl = e.p(L.e_floss);
  R* force = e.p(L.e_force);
  R* act = e.p(L.scratch);             // per-row curvature (D or 0); cone rows 0
  R* Hc = e.p(L.scratch) + L.me;   // per-contact cone Hessian blocks, 36 each
  const int* eint = e.pi(L.e_int);
  const int* cint = e.pi(L.c_int);
  R cost = 0;
  int nsimple = m.nfl;
  // simple rows up to the first contact row
  int first_contact_row = nefc;
  B2S_LOOP
  for (int c = 0; c < ncon; c++) { int a = cint[5 * c + 3]; if (a >= 0) { first_contact_row = a; break; } }
  (void)nsimple;
  B2S_LOOP
  for (int r = lane; r < first_contact_row; r += 32) {
    int type = eint[r] & 255;
    R x = jar[r], D = eD[r], a = 0, f;
    if (type == C_FRICTION) {
      R fl = efl[r], Rr = eR[r];
      if (x <= -Rr * fl) { f = fl; cost += -R(0.5) * Rr * fl * fl - fl * x; }
      else if (x >= Rr * fl) { f = -fl; cost += -R(0.5) * Rr * fl * fl + fl * x; }
      else { f = -D * x; cost += R(0.5) * D * x * x; a = D; }
    } else {
      if (x < 0) { f = -D * x; cost += R(0.5) * D * x * x; a = D; }
      else f = 0;
    }
    force[r] = f;
    if (hess) act[r] = a;
  }
  const R* cfric = e.p(L.c_fric);
  B2S_LOOP
  for (int c = lane; c < ncon; c += 32) {
    int adr = cint[5 * c + 3];
    if (adr < 0) continue;
    int dim = cint[5 * c + 2];
    if (dim == 1) {
      R x = jar[adr], D = eD[adr];
      if (x < 0) { force[adr] = -D * x; cost += R(0.5) * D * x * x; if (hess) act[adr] = D; }
      else { force[adr] = 0; if (hess) act[adr] = 0; }
      if (hess) Hc[m.hc_stride * c] = -1;
      continue;
    }
    R mu = efl[adr], U[6], fr[6];
    fr[0] = mu;
    U[0] = jar[adr] * mu;
    R TT = 0;
    B2S_LOOP
    for (int k = 1; k < dim; k++) { fr[k] = row_friction(cfric + 3 * c, k); U[k] = jar[adr + k] * fr[k]; TT += U[k] * U[k]; }
    R N = U[0], T = r_sqrt(TT);
    if (N >= mu * T || (T <= 0 && N >= 0)) {
      B2S_LOOP
      for (int k = 0; k < dim; k++) { force[adr + k] = 0; if (hess) act[adr + k] = 0; }
      if (hess) Hc[m.hc_stride * c] = -1;
    } else if (mu * N + T <= 0 || (T <= 0 && N < 0)) {
      B2S_LOOP
      for (int k = 0; k < dim; k++) {
        R Dk = eD[adr + k], x = jar[adr + k];
        force[adr + k] = -Dk * x;
        cost += R(0.5) * Dk * x * x;
        if (hess) act[adr + k] = Dk;
      }
      if (hess) Hc[m.hc_stride * c] = -1;
    } else {
      R Dm = eD[adr] / r_max(mu * mu * (1 + mu * mu), Lim<R>::minval());
      R NT = N - mu * T;
      cost += R(0.5) * Dm * NT * NT;
      R f0 = -Dm * NT * mu;
      force[adr] = f0;
      B2S_LOOP
      for (int k = 1; k < dim; k++) force[adr + k] = -f0 / T * U[k] * fr[k];
      if (hess) {
        B2S_LOOP
        for (int k = 0; k < dim; k++) act[adr + k] = 0;
        R* h = Hc + m.hc_stride * c;
        R invT = R(1) / T;
        h[0] = Dm * fr[0] * fr[0];
        B2S_LOOP
        for (int k = 1; k < dim; k++) h[k] = h[k * dim] = -Dm * mu * U[k] * invT * fr[0] * fr[k];
        B2S_LOOP
        for (int a = 1; a < dim; a++)
          B2S_LOOP
          for (int b = 1; b < dim; b++) {
            R v = Dm * mu * mu * U[a] * U[b] * invT * invT - Dm * NT * mu * ((a == b ? invT : R(0)) - U[a] * U[b] * invT * invT * invT);
            h[a * dim + b] = v * fr[a] * fr[b];
          }
      }
    }
  }
  cost = warp_sum(cost);
  __syncwarp();
  return cost;
}

// first / second derivative of the cost along the search direction at step alpha (warp-uniform result)
template <typename R>
DEVN void ls_eval(Eng<R> e, int nefc, int ncon, int first_contact_row, R alpha, R quad1, R quad2, R& d1, R& d2) {
  const DModel<R>& m = e.model();
  const WSLayout& L = e.lay();
  int lane = e.lane;
  const R* jar = e.p(L.e_jar); const R* jv = e.p(L.e_jv); const R* eD = e.p(L.e_D); const R* eR = e.p(L.e_R);
  const R* efl = e.p(L.e_floss);
  const int* eint = e.pi(L.e_int); const int* cint = e.pi(L.c_int);
  const R* cfric = e.p(L.c_fric);
  R g = 0, h = 0;
  B2S_LOOP
  for (int r = lane; r < first_contact_row; r += 32) {
    R x = jar[r] + alpha * jv[r], v = jv[r], D = eD[r];
    if ((eint[r] & 255) == C_FRICTION) {
      R fl = efl[r], Rr = eR[r];
      if (x <= -Rr * fl) g += -fl * v;
      else if (x >= Rr * fl) g += fl * v;
      else { g += D * x * v; h += D * v * v; }
    } else if (x < 0) { g += D * x * v; h += D * v * v; }
  }
  B2S_LOOP
  for (int c = lane; c < ncon; c += 32) {
    int adr = cint[5 * c + 3];
    if (adr < 0) continue;
    int dim = cint[5 * c + 2];
    R x0 = jar[adr] + alpha * jv[adr], v0 = jv[adr];
    if (dim == 1) { if (x0 < 0) { g += eD[adr] * x0 * v0; h += eD[adr] * v0 * v0; } continue; }
    R mu = efl[adr];
    R N = x0 * mu, Nd = v0 * mu, TT = 0, UV = 0, VV = 0;
    B2S_LOOP
    for (int k = 1; k < dim; k++) {
      R fk = row_friction(cfric + 3 * c, k);
      R u = (jar[adr + k] + alpha * jv[adr + k]) * fk, w = jv[adr + k] * fk;
      TT += u * u; UV += u * w; VV += w * w;
    }
    R T = r_sqrt(TT);
    if (N >= mu * T || (T <= 0 && N >= 0)) {
    } else if (mu * N + T <= 0 || (T <= 0 && N < 0)) {
      B2S_LOOP
      for (int k = 0; k < dim; k++) {
        R xk = jar[adr + k] + alpha * jv[adr + k], vk = jv[adr + k], Dk = eD[adr + k];
        g += Dk * xk * vk; h += Dk * vk * vk;
      }
    } else {
      R Dm = eD[adr] / r_max(mu * mu * (1 + mu * mu), Lim<R>::minval());
      R NT = N - mu * T;
      R Td = UV / T, Tdd = VV / T - UV * UV / (T * T * T);
      R NTd = Nd - mu * Td;
      g += Dm * NT * NTd;
      h += Dm * (NTd * NTd + NT * (-mu * Tdd));
    }
  }
  d1 = quad1 + alpha * quad2 + warp_sum(g);
  d2 = quad2 + warp_sum(h);
}

// Newton solve: qacc (workspace) <- argmin; efc_force, qfrc_constraint filled.  Returns iterations used.
template <typename R> DEVN int solve(Eng<R> e, int nefc, int ncon, int& warn) {
  const DModel<R>& m = e.model();
  const WSLayout& L = e.lay();
  int lane = e.lane, nv = m.nv;
  R* qacc = e.p(L.qacc); R* qcon = e.p(L.qcon);
  const R* qs = e.p(L.qsmooth); const R* qas = e.p(L.qaccs);
  if (nefc == 0) {
    B2S_LOOP
    for (int i = lane; i < nv; i += 32) { qacc[i] = qas[i]; qcon[i] = 0; }
    __syncwarp();
    return 0;
  }
  const R* M = e.p(L.M); R* H = e.p(L.H); const R* J = e.p(L.J);
  R* jar = e.p(L.e_jar); R* jv = e.p(L.e_jv); R* force = e.p(L.e_force); const R* aref = e.p(L.e_aref);
  R* Ma = e.p(L.Ma); R* grad = e.p(L.grad); R* search = e.p(L.search); R* Mv = e.p(L.Mv);
  const int* cint = e.pi(L.c_int);
  const int* eint = e.pi(L.e_int);
  R* act = e.p(L.scratch); R* Hcb = e.p(L.scratch) + L.me;
  R scale = R(1) / (meaninertia_of(m, e.state(), e.env) * R(nv > 1 ? nv : 1));
  int first_contact_row = nefc;
  B2S_LOOP
  for (int c = 0; c < ncon; c++) { int a = cint[5 * c + 3]; if (a >= 0) { first_contact_row = a; break; } }
  // does any constraint couple two different moving trees?  (then the Hessian is not block diagonal)
  bool cross_tree = false;
  B2S_LOOP
  for (int c = 0; c < ncon; c++) {
    if (cint[5 * c + 3] < 0) continue;
    int t1 = m.body_treeid[m.geom_bodyid[cint[5 * c]]], t2 = m.body_treeid[m.geom_bodyid[cint[5 * c + 1]]];
    if (t1 >= 0 && t2 >= 0 && t1 != t2) cross_tree = true;
  }
  // both limit rows of one joint (a range narrower than twice its margin) follow each other and hit one dof
  bool two_sided = false;
  B2S_LOOP
  for (int r = lane + 1; r < first_contact_row; r += 32) two_sided |= (eint[r] & 255) == C_LIMIT && eint[r - 1] == eint[r];
  two_sided = __any_sync(B2S_FULL, two_sided);

  // --- warm start: previous qacc unless the unconstrained acceleration is cheaper
  R cost_ws = 0, cost_sm = 0;
  B2S_LOOP
  for (int pass = 0; pass < 2; pass++) {
    const R* q = pass == 0 ? e.p(L.qacc_ws) : qas;
    B2S_LOOP
    for (int r = lane; r < nefc; r += 32) {
      R s = -aref[r];
      B2S_LOOP
      for (int k = 0; k < nv; k++) s += J[r * nv + k] * q[k];
      jar[r] = s;
    }
    __syncwarp();
    R cc = constraint_update(e, nefc, ncon, false);
    if (pass == 0) {
      R gs = 0;
      B2S_LOOP
      for (int i = lane; i < nv; i += 32) {
        R s = 0;
        B2S_LOOP
        for (int k = 0; k < nv; k++) s += M[i * nv + k] * q[k];
        gs += R(0.5) * (s - qs[i]) * (q[i] - qas[i]);
      }
      cost_ws = cc + warp_sum(gs);
    } else cost_sm = cc;
  }
  {
    const R* q = cost_ws < cost_sm ? e.p(L.qacc_ws) : qas;
    B2S_LOOP
    for (int i = lane; i < nv; i += 32) qacc[i] = q[i];
  }
  __syncwarp();
  R prev_cost = 0;
  int niter = 0;
#ifdef B2S_INSTR
  int instr_ls = 0;
#define INSTR_SOLVE_DONE { const DState<R>& st_ = e.state(); if (lane == 0 && st_.stats) { atomicAdd(st_.stats + min(niter, 15), 1); atomicAdd(st_.stats + 16, instr_ls); atomicAdd(st_.stats + 17, 1); } \
                           if (lane == 0 && st_.solve_ls) st_.solve_ls[e.env] = instr_ls; }
#else
#define INSTR_SOLVE_DONE
#endif
  // Ma = M qacc and jar = J qacc - aref are formed once and then moved along the search direction with the step
  // (Ma += alpha Mv, jar += alpha jv), as the reference engine does
  B2S_LOOP
  for (int i = lane; i < nv; i += 32) {
    R s = 0;
    B2S_LOOP
    for (int k = 0; k < nv; k++) s += M[i * nv + k] * qacc[k];
    Ma[i] = s;
  }
  B2S_LOOP
  for (int r = lane; r < nefc; r += 32) {
    R s = -aref[r];
    B2S_LOOP
    for (int k = 0; k < nv; k++) s += J[r * nv + k] * qacc[k];
    jar[r] = s;
  }
  __syncwarp();
  bool stale = false;  // efc_force older than jar?
  B2S_LOOP
  for (int iter = 0; iter <= m.iterations; iter++) {
    R cost = constraint_update(e, nefc, ncon, true);
    stale = false;
    R gs = 0, gn = 0;
    B2S_LOOP
    for (int i = lane; i < nv; i += 32) gs += R(0.5) * (Ma[i] - qs[i]) * (qacc[i] - qas[i]);
    cost += warp_sum(gs);
    B2S_LOOP
    for (int i = lane; i < nv; i += 32) {
      R s = Ma[i] - qs[i];
      B2S_LOOP
      for (int r = 0; r < nefc; r++) s -= J[r * nv + i] * force[r];
      grad[i] = s;
      gn += s * s;
    }
    R gnorm = r_sqrt(warp_sum(gn));
    __syncwarp();
    // fp32 as fp64: the solve stops on the tolerance alone.  An extra exit at the rounding noise of the cost (16 eps |cost|) ended
    // stiff multi-contact solves early - a nut squeezed between two fingers then turned by a large angle within one substep
    if (iter > 0) {
      R improvement = scale * (prev_cost - cost);
      if (improvement < m.tolerance || scale * gnorm < m.tolerance) break;
    } else if (scale * gnorm < m.tolerance) break;
    if (iter == m.iterations) break;
    prev_cost = cost;
    niter = iter + 1;
    // --- Hessian H = M + J^T act J + cone blocks, exploiting row structure:
    //   friction-loss / limit rows are +-unit vectors -> diagonal terms only;
    //   a contact's rows touch only the dofs that move exactly one of its two bodies -> entries on that support only
    B2S_LOOP
    for (int k = lane; k < nv * nv; k += 32) H[k] = M[k];
    __syncwarp();
    // a dof can carry a friction-loss row AND the lower and upper limit rows of its joint: one pass of plain adds per kind (rows of
    // one kind hit distinct dofs) keeps the summation order fixed - a float atomicAdd left it to the hardware, and two handles
    // stepping side by side then drifted apart.  Pass 0: friction loss, pass 1: limits, pass 2: the upper side of a two-sided joint
    B2S_LOOP
    for (int pass = 0; pass < (two_sided ? 3 : 2); pass++) {
      B2S_LOOP
      for (int r = lane; r < first_contact_row; r += 32) {
        int ty = eint[r] & 255, id = eint[r] >> 8;
        R d = act[r];
        int p = ty == C_FRICTION ? 0 : (two_sided && r > 0 && eint[r - 1] == eint[r] ? 2 : 1);
        if (p == pass && d != 0) {
          int dof = ty == C_FRICTION ? id : m.jnt_dofadr[id];
          H[dof * nv + dof] += d;
        }
      }
      __syncwarp();
    }
    {
      int* dofs = reinterpret_cast<int*>(Hcb + m.hc_stride * L.mc);
      B2S_LOOP
      for (int c = 0; c < ncon; c++) {
        int adr = cint[5 * c + 3];
        if (adr < 0) continue;
        int dim = cint[5 * c + 2];
        const R* h = Hcb + m.hc_stride * c;
        bool cone = h[0] >= 0;
        bool any = cone;
        B2S_LOOP
        for (int k = 0; k < dim && !any; k++) any = act[adr + k] != 0;
        if (!any) continue;
        unsigned long long mask = m.body_dofmask[m.geom_bodyid[cint[5 * c]]] ^ m.body_dofmask[m.geom_bodyid[cint[5 * c + 1]]];
        int ns = __popcll(mask);
        B2S_LOOP
        for (int i = lane; i < nv; i += 32)
          if ((mask >> i) & 1ull) dofs[__popcll(mask & ((1ull << i) - 1ull))] = i;
        __syncwarp();
        int ne = ns * (ns + 1) / 2;
        B2S_LOOP
        for (int w = lane; w < ne; w += 32) {
          int ia = (int)((r_sqrt(R(8 * w + 1)) - R(1)) * R(0.5));
          while ((ia + 1) * (ia + 2) / 2 <= w) ia++;
          while (ia * (ia + 1) / 2 > w) ia--;
          int ib = w - ia * (ia + 1) / 2;
          int a = dofs[ia], b = dofs[ib];
          R sacc = 0;
          if (cone) {
            B2S_LOOP
            for (int x = 0; x < dim; x++) {
              R t = 0;
              B2S_LOOP
              for (int y = 0; y < dim; y++) t += h[x * dim + y] * J[(adr + y) * nv + b];
              sacc += J[(adr + x) * nv + a] * t;
            }
          } else {
            B2S_LOOP
            for (int k = 0; k < dim; k++) sacc += act[adr + k] * J[(adr + k) * nv + a] * J[(adr + k) * nv + b];
          }
          H[a * nv + b] += sacc;
          if (a != b) H[b * nv + a] += sacc;
        }
        __syncwarp();
      }
    }
    B2S_LOOP
    for (int i = lane; i < nv; i += 32) search[i] = -grad[i];
    __syncwarp();
    if (e.spd_solve(H, nv, (const R*)nullptr, R(0), search, H, !cross_tree)) { warn |= 16; break; }
    // --- exact line search
    R q1 = 0, q2 = 0;
    B2S_LOOP
    for (int i = lane; i < nv; i += 32) {
      R s = 0;
      B2S_LOOP
      for (int k = 0; k < nv; k++) s += M[i * nv + k] * search[k];
      Mv[i] = s;
      q1 += search[i] * (Ma[i] - qs[i]);
      q2 += search[i] * s;
    }
    R quad1 = warp_sum(q1), quad2 = warp_sum(q2);
    B2S_LOOP
    for (int r = lane; r < nefc; r += 32) {
      R s = 0;
      B2S_LOOP
      for (int k = 0; k < nv; k++) s += J[r * nv + k] * search[k];
      jv[r] = s;
    }
    __syncwarp();
    R d1, d2, alpha = 0, lo = 0, hi = -1;
    ls_eval(e, nefc, ncon, first_contact_row, R(0), quad1, quad2, d1, d2);
    if (d1 >= 0) break;
    // Newton decrement: -d1(0) = grad^T H^-1 grad.  When half of it is below the stopping tolerance this step is the
    // last one: take it and skip the iteration that would only confirm convergence.
    bool last = R(0.5) * scale * (-d1) < m.tolerance;
    R gtol = (sizeof(R) == 4 ? R(1e-3) : R(1e-12)) * r_abs(d1);
    alpha = -d1 / d2;
    B2S_LOOP
    for (int ls = 0; ls < (sizeof(R) == 4 ? 20 : 100); ls++) {
      ls_eval(e, nefc, ncon, first_contact_row, alpha, quad1, quad2, d1, d2);
#ifdef B2S_INSTR
      instr_ls++;
#endif
      if (r_abs(d1) <= gtol) break;
      if (d1 < 0) lo = alpha; else hi = alpha;
      R next = alpha - d1 / d2;
      if (hi < 0) { if (next <= lo) next = 2 * alpha + R(1e-12); }
      else if (next <= lo || next >= hi) next = R(0.5) * (lo + hi);
      if (hi >= 0 && hi - lo < (sizeof(R) == 4 ? R(1e-7) : R(1e-15)) * r_max(R(1), hi)) break;
      alpha = next;
    }
    B2S_LOOP
    for (int i = lane; i < nv; i += 32) { qacc[i] += alpha * search[i]; Ma[i] += alpha * Mv[i]; }
    B2S_LOOP
    for (int r = lane; r < nefc; r += 32) jar[r] += alpha * jv[r];
    stale = true;
    __syncwarp();
    if (last) break;
  }
  // --- final forces at the solution
  if (stale) constraint_update(e, nefc, ncon, false);
  B2S_LOOP
  for (int i = lane; i < nv; i += 32) {
    R s = 0;
    B2S_LOOP
    for (int r = 0; r < nefc; r++) s += J[r * nv + i] * force[r];
    qcon[i] = s;
  }
  __syncwarp();
  INSTR_SOLVE_DONE
  return niter;
}
