// Fused controller: OSC_POSE arm + GRIP gripper evaluated by the owning warp between step1 and step2 of every
// substep (no HBM round trip).  Reference semantics, file:line -
//   OperationalSpaceController.set_goal / run_controller   robosuite/controllers/parts/arm/osc.py:225-283, 403-495
//   opspace_matrices / nullspace_torques / orientation_error  robosuite/utils/control_utils.py:7-111
//   Controller.scale_action                                 robosuite/controllers/parts/controller.py:149-168
//   PandaGripper.format_action                              robosuite/models/grippers/panda_gripper.py:43-58
//   SimpleGripController.run_controller                     robosuite/controllers/parts/gripper/simple_grip.py:150-186
//   FixedBaseRobot.control (clip to ctrlrange)              robosuite/robots/fixed_base_robot.py:149-153
#pragma once
#include "b2s_solver.cuh"
#include "b2s_oscmath.h"

// small dense algebra of the controller runs in CA (double keeps Lambda = (J M^-1 J^T)^-1 well conditioned even
// when the arm is near a singular pose; the blocks are 7x7 / 6x6 so the cost is negligible).  The operational-space inverses
// keep numpy's pinv meaning (control_utils.py:74-76) with b2s_oscmath.h's tests: Cholesky / closed form far from the cut-off,
// the Jacobi pseudo-inverse near it.
typedef double CA;

template <typename R> struct CtrlState {
  R goal_pos[3], goal_ori[9], grip[4];
};

template <typename R> DEV void ctrl_load(Eng<R> e, CtrlState<R>& cs, int env) {
  const DState<R>& s = e.state();
  size_t E = env;
  for (int k = 0; k < 3; k++) cs.goal_pos[k] = s.goal_pos[E * 3 + k];
  for (int k = 0; k < 9; k++) cs.goal_ori[k] = s.goal_ori[E * 9 + k];
  for (int k = 0; k < 4; k++) cs.grip[k] = s.grip_state[E * 4 + k];
}
template <typename R> DEV void ctrl_store(Eng<R> e, CtrlState<R>& cs, int env) {
  const DState<R>& s = e.state();
  size_t E = env;
  if (e.lane == 0) {
    for (int k = 0; k < 3; k++) s.goal_pos[E * 3 + k] = cs.goal_pos[k];
    for (int k = 0; k < 9; k++) s.goal_ori[E * 9 + k] = cs.goal_ori[k];
    for (int k = 0; k < 4; k++) s.grip_state[E * 4 + k] = cs.grip[k];
  }
}

// rotation matrix of a scaled axis-angle vector, rounded through float32 like the reference
// (transform_utils.py:461-487, 515-538)
template <typename R> DEV void delta_rotmat(R* Rm, const R* aa) {
  double angle = sqrt((double)aa[0] * aa[0] + (double)aa[1] * aa[1] + (double)aa[2] * aa[2]);
  double qd[4] = {0, 0, 0, 1};
  if (angle != 0.0) {
    double sn = sin(angle / 2.0);
    qd[0] = aa[0] / angle * sn; qd[1] = aa[1] / angle * sn; qd[2] = aa[2] / angle * sn; qd[3] = cos(angle / 2.0);
  }
  float q[4] = {(float)qd[3], (float)qd[0], (float)qd[1], (float)qd[2]};
  float n = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
  if (n < 8.881784197001252e-16f) { for (int i = 0; i < 9; i++) Rm[i] = (i % 4 == 0); return; }
  float rr = 2.0f / n;
  float sc = (float)sqrt((double)rr);
  for (int i = 0; i < 4; i++) q[i] *= sc;
#define Q2(i, j) (q[i] * q[j])
  Rm[0] = 1.0f - Q2(2, 2) - Q2(3, 3); Rm[1] = Q2(1, 2) - Q2(3, 0); Rm[2] = Q2(1, 3) + Q2(2, 0);
  Rm[3] = Q2(1, 2) + Q2(3, 0); Rm[4] = 1.0f - Q2(1, 1) - Q2(3, 3); Rm[5] = Q2(2, 3) - Q2(1, 0);
  Rm[6] = Q2(1, 3) - Q2(2, 0); Rm[7] = Q2(2, 3) + Q2(1, 0); Rm[8] = 1.0f - Q2(1, 1) - Q2(2, 2);
#undef Q2
}

// JointVelocityController (robosuite/controllers/parts/generic/joint_vel.py:129-209): PID on joint velocity with a
// 5-sample derivative ring, anti-windup, + qfrc_bias; the constructor line :127 (assignment to a read-only property)
// is read as the sibling controllers spell it (`use_torque_compensation`, joint_tor.py:109).  One lane per joint.
// JointPositionController (joint_pos.py:160-262; kind 3: goal_qpos = q + scaled delta at policy steps, torque =
// M_arm (kp e - kd qvel) + qfrc_bias) and JointTorqueController (joint_tor.py:112-160; kind 4: goal torque = clipped scaled
// action, torque = goal + qfrc_bias).  One lane per joint; the goal lives in the first 8 words of the jv_state row.
template <typename R>
DEVN void ctrl_run_joint(Eng<R> e, CtrlState<R>& cs, int env, const R* action) {
  const DModel<R>& m = e.model();
  const WSLayout& L = e.lay();
  const DState<R>& s = e.state();
  const CtrlCfgDev& cc = e.ccfg();
  int lane = e.lane, na = cc.n_arm, nv = m.nv;
  R* st = s.jv_state + (size_t)env * 72;
  R* ctrl = e.p(L.ctrl);
  int k = lane < na ? lane : 0, dof = cc.arm_dof[k], u = cc.arm_act[k];
  const int off = cc.imp ? cc.imp->off : 0;  // variable impedance: the delta follows the gains
  const size_t G = (size_t)env * 16;  // this environment's gain row
  R goal = st[k];
  if (action && lane < na) {
    if (cc.gain) imp_gain(cc.imp, action + (size_t)env * cc.action_dim, k, cc.gain + G + k, cc.gain + G + 8 + k);  // before the goal
    R a = r_clamp(action[(size_t)env * cc.action_dim + off + k], (R)cc.jv_in_min[k], (R)cc.jv_in_max[k]);
    R scale = (R)(fabs(cc.jv_out_max[k] - cc.jv_out_min[k]) / fabs(cc.jv_in_max[k] - cc.jv_in_min[k]));
    R sc = (a - (R)(0.5 * (cc.jv_in_max[k] + cc.jv_in_min[k]))) * scale + (R)(0.5 * (cc.jv_out_max[k] + cc.jv_out_min[k]));
    goal = cc.kind == 3 ? e.p(L.qpos)[cc.arm_qpos[k]] + sc : r_clamp(sc, m.act_ctrlrange[2 * u], m.act_ctrlrange[2 * u + 1]);
    st[k] = goal;
  }
  R tau;
  if (cc.kind == 3) {
    R kp = (R)cc.jv_kp[k], kd = (R)cc.jv_kd[k];
    if (cc.gain) { kp = (R)cc.gain[G + k]; kd = (R)cc.gain[G + 8 + k]; }
    R des = lane < na ? (goal - e.p(L.qpos)[cc.arm_qpos[k]]) * kp - e.p(L.qvel)[dof] * kd : R(0);
    tau = 0;
    for (int b = 0; b < na; b++) {
      R db = __shfl_sync(B2S_FULL, des, b);
      tau += e.p(L.M)[dof * nv + cc.arm_dof[b]] * db;
    }
    tau = cc.jv_torque_comp ? tau + e.p(L.bias)[dof] : des;
  } else {
    tau = goal + (cc.jv_torque_comp ? e.p(L.bias)[dof] : R(0));
  }
  if (lane < na) {
    s.ctrl_torque[(size_t)env * 8 + k] = tau;
    ctrl[u] = r_clamp(tau, m.act_ctrlrange[2 * u], m.act_ctrlrange[2 * u + 1]);
  }
  if (action) {
    R ga = action[(size_t)env * cc.action_dim + off + na];
    R sg = ga > 0 ? R(1) : (ga < 0 ? R(-1) : R(0));
    for (int g = 0; g < cc.n_grip; g++) cs.grip[g] = r_clamp(cs.grip[g] + (R)(cc.grip_sign[g] * cc.grip_speed) * sg, R(-1), R(1));
  }
  if (lane < cc.n_grip) {
    int ug = cc.grip_act[lane];
    R lo = m.act_ctrlrange[2 * ug], hi = m.act_ctrlrange[2 * ug + 1];
    ctrl[ug] = r_clamp(R(0.5) * (hi + lo) + R(0.5) * (hi - lo) * cs.grip[lane], lo, hi);
  }
  __syncwarp();
}

template <typename R>
DEVN void ctrl_run_jv(Eng<R> e, CtrlState<R>& cs, int env, const R* action) {
  const DModel<R>& m = e.model();
  const WSLayout& L = e.lay();
  const DState<R>& s = e.state();
  const CtrlCfgDev& cc = e.ccfg();
  int lane = e.lane, na = cc.n_arm;
  R* st = s.jv_state + (size_t)env * 72;
  R* ctrl = e.p(L.ctrl);
  int ptr = (int)st[64], size = (int)st[65];
  bool saturated = st[66] != 0;
  ptr = (ptr + 1) % 5;
  if (size < 5) size++;
  R diff = 0;
  if (lane < na) {
    int k = lane, dof = cc.arm_dof[k];
    R goal = st[k];
    if (action) {
      R a = r_clamp(action[(size_t)env * cc.action_dim + k], (R)cc.jv_in_min[k], (R)cc.jv_in_max[k]);
      R scale = (R)(fabs(cc.jv_out_max[k] - cc.jv_out_min[k]) / fabs(cc.jv_in_max[k] - cc.jv_in_min[k]));
      goal = (a - (R)(0.5 * (cc.jv_in_max[k] + cc.jv_in_min[k]))) * scale + (R)(0.5 * (cc.jv_out_max[k] + cc.jv_out_min[k]));
      if (cc.jv_use_vel_limits) goal = r_clamp(goal, (R)cc.jv_vel_lo, (R)cc.jv_vel_hi);
      st[k] = goal;
    }
    R err = goal - e.p(L.qvel)[dof];
    st[24 + 8 * ptr + k] = err - st[8 + k];
    st[8 + k] = err;
    R summed = st[16 + k];
    if (!saturated) { summed += err; st[16 + k] = summed; }
    R avg = 0;
    for (int r = 0; r < size; r++) avg += st[24 + 8 * r + k];
    avg /= R(size);
    R tau = (R)cc.jv_kp[k] * err + (R)cc.jv_ki[k] * summed + (R)cc.jv_kd[k] * avg;
    if (cc.jv_torque_comp) tau += e.p(L.bias)[dof];
    int u = cc.arm_act[k];
    R cl = r_clamp(tau, m.act_ctrlrange[2 * u], m.act_ctrlrange[2 * u + 1]);
    s.ctrl_torque[(size_t)env * 8 + k] = tau;
    ctrl[u] = cl;
    diff = r_abs(cl - tau);
  }
  diff = warp_sum(diff);
  if (action) {
    R ga = action[(size_t)env * cc.action_dim + na];
    R sg = ga > 0 ? R(1) : (ga < 0 ? R(-1) : R(0));
    for (int g = 0; g < cc.n_grip; g++) cs.grip[g] = r_clamp(cs.grip[g] + (R)(cc.grip_sign[g] * cc.grip_speed) * sg, R(-1), R(1));
  }
  if (lane < cc.n_grip) {
    int u = cc.grip_act[lane];
    R lo = m.act_ctrlrange[2 * u], hi = m.act_ctrlrange[2 * u + 1];
    ctrl[u] = r_clamp(R(0.5) * (hi + lo) + R(0.5) * (hi - lo) * cs.grip[lane], lo, hi);
  }
  if (lane == 0) { st[64] = R(ptr); st[65] = R(size); st[66] = diff != 0 ? R(1) : R(0); }
  __syncwarp();
}

template <typename R>
DEVN void ctrl_run(Eng<R> e, CtrlState<R>& cs, int env, const R* action) {
  const DModel<R>& m = e.model();
  const WSLayout& L = e.lay();
  const DState<R>& s = e.state();
  const CtrlCfgDev& cc = e.ccfg();
  if (cc.kind == 2) { ctrl_run_jv(e, cs, env, action); return; }
  if (cc.kind == 3 || cc.kind == 4) { ctrl_run_joint(e, cs, env, action); return; }
  bool policy_step = action != nullptr;
  int lane = e.lane, nv = m.nv, na = cc.n_arm;
  const R* ref_pos = e.p(L.spos) + 3 * cc.eef_site; const R* ref_ori = e.p(L.smat) + 9 * cc.eef_site;
  const R* org_pos = e.p(L.spos) + 3 * cc.base_site; const R* org_ori = e.p(L.smat) + 9 * cc.base_site;
  const size_t G = (size_t)env * 16;  // this environment's gain row (variable impedance)
  if (policy_step) {
    const R* act = action + (size_t)env * cc.action_dim;
    if (cc.gain && lane < 6) imp_gain(cc.imp, act, lane, cc.gain + G + lane, cc.gain + G + 8 + lane);  // before the goal, as set_goal
    if (cc.imp) act += cc.imp->off;  // the delta follows the gains
    const int od = cc.kind == 5 ? 3 : 6;  // OSC_POSITION (osc.py:152-166, 259-270): 3-dim arm action, zero orientation delta
    R sd[6] = {0, 0, 0, 0, 0, 0};
    for (int k = 0; k < od; k++) {
      R a = r_clamp(act[k], (R)cc.input_min[k], (R)cc.input_max[k]);
      R scale = (R)(fabs(cc.output_max[k] - cc.output_min[k]) / fabs(cc.input_max[k] - cc.input_min[k]));
      sd[k] = (a - (R)(0.5 * (cc.input_max[k] + cc.input_min[k]))) * scale + (R)(0.5 * (cc.output_max[k] + cc.output_min[k]));
    }
    R rel[3], inb[3], cur[9], Rd[9];
    v3sub(rel, ref_pos, org_pos);
    m3mulTv(inb, org_ori, rel);
    for (int k = 0; k < 3; k++) cs.goal_pos[k] = inb[k] + sd[k];
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) cur[3 * i + j] = org_ori[i] * ref_ori[j] + org_ori[3 + i] * ref_ori[3 + j] + org_ori[6 + i] * ref_ori[6 + j];
    delta_rotmat(Rd, sd + 3);
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) cs.goal_ori[3 * i + j] = Rd[3 * i] * cur[j] + Rd[3 * i + 1] * cur[3 + j] + Rd[3 * i + 2] * cur[6 + j];
    R ga = act[od];
    R sg = ga > 0 ? R(1) : (ga < 0 ? R(-1) : R(0));
    for (int g = 0; g < cc.n_grip; g++) cs.grip[g] = r_clamp(cs.grip[g] + (R)(cc.grip_sign[g] * cc.grip_speed) * sg, R(-1), R(1));
  }
  // ---- workspace in scratch (CA units)
  CA* sc = reinterpret_cast<CA*>(e.p(L.scratch));
  CA* Jm = sc;            // 6 x na
  CA* Mm = Jm + 48;       // na x na (kept)
  CA* Lc = Mm + 64;       // Cholesky factor of Mm
  CA* X = Lc + 64;        // na x 6 : L^-1 J^T, then M^-1 J^T
  CA* Lf = X + 48;        // 6 x 6 lambda_full (inverse, then lambda)
  CA* Lw = Lf + 36;       // 6 x 6 work (Cholesky of lambda_full_inv)
  CA* vec = Lw + 36;      // F[6] W[6] pt[8] ptm[8] y[6] z[6]
  CA* F = vec; CA* W = vec + 6; CA* pt = vec + 12; CA* ptm = vec + 20; CA* y6 = vec + 28; CA* z6 = vec + 34;
  const R* cdof = e.p(L.cdof); const R* M = e.p(L.M); const R* cvel = e.p(L.cvel);
  int eb = m.site_bodyid[cc.eef_site], bb = m.site_bodyid[cc.base_site];
  unsigned long long emask = m.body_dofmask[eb];
  for (int w = lane; w < 6 * na; w += 32) {
    int r = w / na, k = w % na, i = cc.arm_dof[k];
    CA v = 0;
    if ((emask >> i) & 1ull) {
      const R* cd = cdof + 6 * i;
      if (r < 3) {
        R t[3];
        v3cross(t, cd, ref_pos);
        v = (CA)(cd[3 + r] + t[r]);
      } else v = (CA)cd[r - 3];
    }
    Jm[r * na + k] = v;
  }
  for (int w = lane; w < na * na; w += 32) {
    int a = w / na, b = w % na;
    CA v = (CA)M[cc.arm_dof[a] * nv + cc.arm_dof[b]];
    Mm[w] = v;
    Lc[w] = v;
  }
  // desired wrench (every lane computes the same 6 numbers; lane 0 stores)
  {
    R des_pos[3], des_ori[9], err[6], e3[3] = {0, 0, 0};
    m3mulv(des_pos, org_ori, cs.goal_pos);
    v3add(des_pos, des_pos, org_pos);
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) des_ori[3 * i + j] = org_ori[3 * i] * cs.goal_ori[j] + org_ori[3 * i + 1] * cs.goal_ori[3 + j] + org_ori[3 * i + 2] * cs.goal_ori[6 + j];
    v3sub(err, des_pos, ref_pos);
    for (int col = 0; col < 3; col++) {
      R rc[3] = {ref_ori[col], ref_ori[3 + col], ref_ori[6 + col]}, rd[3] = {des_ori[col], des_ori[3 + col], des_ori[6 + col]}, cr[3];
      v3cross(cr, rc, rd);
      v3add(e3, e3, cr);
    }
    for (int k = 0; k < 3; k++) err[3 + k] = R(0.5) * e3[k];
    // site velocities from the owning bodies' spatial velocity
    R vel[6], bvel[6], t[3];
    const R* cv = cvel + 6 * eb;
    v3cross(t, cv, ref_pos);
    vel[0] = cv[3] + t[0]; vel[1] = cv[4] + t[1]; vel[2] = cv[5] + t[2]; vel[3] = cv[0]; vel[4] = cv[1]; vel[5] = cv[2];
    const R* bv = cvel + 6 * bb;
    v3cross(t, bv, org_pos);
    bvel[0] = bv[3] + t[0]; bvel[1] = bv[4] + t[1]; bvel[2] = bv[5] + t[2]; bvel[3] = bv[0]; bvel[4] = bv[1]; bvel[5] = bv[2];
    if (lane < 6) {  // this lane wrote its own gains on a policy substep
      const CA kp = cc.gain ? cc.gain[G + lane] : cc.kp[lane], kd = cc.gain ? cc.gain[G + 8 + lane] : cc.kd[lane];
      F[lane] = (CA)err[lane] * kp - ((CA)vel[lane] - (CA)bvel[lane]) * kd;
    }
  }
  __syncwarp();
  // Cholesky of the arm mass matrix (na x na) - column by column, lanes = rows
  for (int j = 0; j < na; j++) {
    if (lane >= j && lane < na) {
      CA sacc = Lc[lane * na + j];
      for (int k = 0; k < j; k++) sacc -= Lc[lane * na + k] * Lc[j * na + k];
      Lc[lane * na + j] = sacc;
    }
    __syncwarp();
    CA d = Lc[j * na + j];
    if (!(d > 1e-300)) d = 1e-300;
    CA inv = rsqrt(d);
    __syncwarp();
    if (lane > j && lane < na) Lc[lane * na + j] *= inv;
    if (lane == j) Lc[j * na + j] = inv;  // the diagonal keeps 1 / l_jj: the triangular solves multiply instead of divide
    __syncwarp();
  }
  // X = L^-1 J^T (lane = column r of J^T), then Y = L^-T X = M^-1 J^T
  if (lane < 6) {
    CA x[8];
    for (int a = 0; a < na; a++) {
      CA sacc = Jm[lane * na + a];
      for (int k = 0; k < a; k++) sacc -= Lc[a * na + k] * x[k];
      x[a] = sacc * Lc[a * na + a];
    }
    for (int a = 0; a < na; a++) X[a * 6 + lane] = x[a];
  }
  __syncwarp();
  // lambda_full_inv = X^T X
  for (int w = lane; w < 36; w += 32) {
    int r = w / 6, q = w % 6;
    CA sacc = 0;
    for (int a = 0; a < na; a++) sacc += X[a * 6 + r] * X[a * 6 + q];
    Lf[w] = sacc;
    Lw[w] = sacc;
  }
  __syncwarp();
  if (lane < 6) {  // back substitution: M^-1 J^T
    CA x[8];
    for (int a = 0; a < na; a++) x[a] = X[a * 6 + lane];
    for (int a = na - 1; a >= 0; a--) {
      CA sacc = x[a];
      for (int k = a + 1; k < na; k++) sacc -= Lc[k * na + a] * x[k];
      x[a] = sacc * Lc[a * na + a];
    }
    for (int a = 0; a < na; a++) X[a * 6 + lane] = x[a];
  }
  // 3x3 blocks -> decoupled wrench (lanes 6 / 7): pinv of the packed block, closed form unless near numpy's cut-off
  if (cc.uncouple && (lane == 6 || lane == 7)) {
    int o = lane == 6 ? 0 : 3;
    const CA blk[6] = {Lf[o * 6 + o], Lf[(o + 1) * 6 + o], Lf[(o + 1) * 6 + o + 1],
                       Lf[(o + 2) * 6 + o], Lf[(o + 2) * 6 + o + 1], Lf[(o + 2) * 6 + o + 2]};
    osc_block3_apply(blk, 0, F + o, W + o);
  }
  __syncwarp();
  // full 6x6: Cholesky of lambda_full_inv in Lw, inverse into Lf (lane = column of the identity).  The smallest pivot over the
  // largest diagonal entry decides, as in osc_torques, whether the matrix may be within pinv's cut-off of singular: then lane 0
  // replaces Lf (still lambda_full_inv) by its Jacobi pseudo-inverse instead.
  CA dmax = 0, pmin = 1e300;
  for (int j = 0; j < 6; j++) dmax = fmax(dmax, Lf[j * 7]);
  for (int j = 0; j < 6; j++) {
    if (lane >= j && lane < 6) {
      CA sacc = Lw[lane * 6 + j];
      for (int k = 0; k < j; k++) sacc -= Lw[lane * 6 + k] * Lw[j * 6 + k];
      Lw[lane * 6 + j] = sacc;
    }
    __syncwarp();
    CA d = Lw[j * 6 + j];
    if (d < pmin) pmin = d;
    if (!(d > 1e-300)) d = 1e-300;
    CA inv = rsqrt(d);
    __syncwarp();
    if (lane > j && lane < 6) Lw[lane * 6 + j] *= inv;
    if (lane == j) Lw[j * 6 + j] = inv;
    __syncwarp();
  }
  if (!(dmax > 0 && pmin / dmax > 1e-11)) {
    if (lane == 0) osc_pinv_sym_jacobi(Lf, 6);
  } else if (lane < 6) {
    CA x[6];
    for (int a = 0; a < 6; a++) {
      CA sacc = a == lane ? 1.0 : 0.0;
      for (int k = 0; k < a; k++) sacc -= Lw[a * 6 + k] * x[k];
      x[a] = sacc * Lw[a * 6 + a];
    }
    for (int a = 5; a >= 0; a--) {
      CA sacc = x[a];
      for (int k = a + 1; k < 6; k++) sacc -= Lw[k * 6 + a] * x[k];
      x[a] = sacc * Lw[a * 6 + a];
    }
    for (int a = 0; a < 6; a++) Lf[a * 6 + lane] = x[a];
  }
  // nullspace posture torque inputs
  if (lane < na) {
    CA kv = 2.0 * sqrt(cc.null_kp);
    pt[lane] = cc.null_kp * ((CA)s.init_qpos_arm[(size_t)env * 8 + lane] - (CA)e.p(L.qpos)[cc.arm_qpos[lane]]) - kv * (CA)e.p(L.qvel)[cc.arm_dof[lane]];
  }
  __syncwarp();
  if (!cc.uncouple && lane < 6) {
    CA sacc = 0;
    for (int q = 0; q < 6; q++) sacc += Lf[lane * 6 + q] * F[q];
    W[lane] = sacc;
  }
  if (lane < na) {
    CA sacc = 0;
    for (int b = 0; b < na; b++) sacc += Mm[lane * na + b] * pt[b];
    ptm[lane] = sacc;
  }
  __syncwarp();
  if (lane < 6) {  // y = (M^-1 J^T)^T ptm
    CA sacc = 0;
    for (int a = 0; a < na; a++) sacc += X[a * 6 + lane] * ptm[a];
    y6[lane] = sacc;
  }
  __syncwarp();
  if (lane < 6) {
    CA sacc = 0;
    for (int q = 0; q < 6; q++) sacc += Lf[lane * 6 + q] * y6[q];
    z6[lane] = sacc;
  }
  __syncwarp();
  R* ctrl = e.p(L.ctrl);
  if (lane < na) {
    CA tau = (CA)e.p(L.bias)[cc.arm_dof[lane]] + ptm[lane];
    for (int r = 0; r < 6; r++) tau += Jm[r * na + lane] * (W[r] - z6[r]);
    int u = cc.arm_act[lane];
    s.ctrl_torque[(size_t)env * 8 + lane] = (R)tau;
    ctrl[u] = r_clamp((R)tau, m.act_ctrlrange[2 * u], m.act_ctrlrange[2 * u + 1]);
  }
  if (lane < cc.n_grip) {
    int u = cc.grip_act[lane];
    R lo = m.act_ctrlrange[2 * u], hi = m.act_ctrlrange[2 * u + 1];
    ctrl[u] = r_clamp(R(0.5) * (hi + lo) + R(0.5) * (hi - lo) * cs.grip[lane], lo, hi);
  }
  __syncwarp();
}

// rotation matrix -> quaternion (w >= 0), same canonical sign as the reference's mat2quat (transform_utils.py:316-356)
template <typename R> DEV void mat2quat_wpos(const R* M, R* q) {
  R tr = M[0] + M[4] + M[8];
  if (tr > 0) {
    R s = r_sqrt(tr + R(1)) * 2;
    q[0] = R(0.25) * s; q[1] = (M[7] - M[5]) / s; q[2] = (M[2] - M[6]) / s; q[3] = (M[3] - M[1]) / s;
  } else if (M[0] > M[4] && M[0] > M[8]) {
    R s = r_sqrt(R(1) + M[0] - M[4] - M[8]) * 2;
    q[0] = (M[7] - M[5]) / s; q[1] = R(0.25) * s; q[2] = (M[1] + M[3]) / s; q[3] = (M[2] + M[6]) / s;
  } else if (M[4] > M[8]) {
    R s = r_sqrt(R(1) + M[4] - M[0] - M[8]) * 2;
    q[0] = (M[2] - M[6]) / s; q[1] = (M[1] + M[3]) / s; q[2] = R(0.25) * s; q[3] = (M[5] + M[7]) / s;
  } else {
    R s = r_sqrt(R(1) + M[8] - M[0] - M[4]) * 2;
    q[0] = (M[3] - M[1]) / s; q[1] = (M[2] + M[6]) / s; q[2] = (M[5] + M[7]) / s; q[3] = R(0.25) * s;
  }
  if (q[0] < 0) { q[0] = -q[0]; q[1] = -q[1]; q[2] = -q[2]; q[3] = -q[3]; }
  qnormalize(q);
}

// Observation row: one table entry per scalar (MujocoEnv._get_observations, environments/base.py:429-465; sensors
// robots/robot.py:347-392,412-484 and the task's object observables e.g. manipulation/lift.py:371-397).
// qpos/qvel/qacc are the freshly integrated values, poses are those of the last step1 (reference staleness).
// one scalar of the observation / task tables; `prev` = this environment's previous observation row (lagged entries)
template <typename R> DEV R table_value(const Eng<R>& e, int op, int a, int b, const R* prev, int fresh) {
  const WSLayout& L = e.lay();
  if (op >= OB_SEL_BODY_POS) {  // the environment's selected object (b2s_obs_objects): the body's plain op
    const CtrlCfgDev& cc = e.ccfg();
    const int k = cc.obj_sel[e.env];
    if (k < 0 || k >= cc.n_sel) { atomicOr(e.state().warn + e.env, 512); return R(0); }  // nothing is read through a bad selection
    if (op == OB_SEL_INDEX) return R(k);
    a = cc.sel_body[k];
    op = op == OB_SEL_BODY_POS ? OB_BODY_POS : OB_BODY_QUAT_XYZW;
  }
  R v = 0;
  switch (op) {
    case OB_QPOS: v = e.p(L.qpos)[a]; break;
    case OB_COS_QPOS: { R sn, cs; r_sincos(e.p(L.qpos)[a], &sn, &cs); v = cs; break; }
    case OB_SIN_QPOS: { R sn, cs; r_sincos(e.p(L.qpos)[a], &sn, &cs); v = sn; break; }
    case OB_QVEL: v = e.p(L.qvel)[a]; break;
    case OB_QACC: v = e.p(L.qacc)[a]; break;
    case OB_SITE_POS: v = e.p(L.spos)[3 * a + b]; break;
    case OB_BODY_POS: v = e.p(L.xpos)[3 * a + b]; break;
    case OB_BODY_QUAT_XYZW: v = e.p(L.xquat)[4 * a + ((b + 1) & 3)]; break;
    case OB_SITE_QUAT_XYZW: { R q[4]; mat2quat_wpos(e.p(L.smat) + 9 * a, q); v = q[(b + 1) & 3]; break; }
    case OB_BODY_MINUS_SITE: v = e.p(L.xpos)[3 * (a >> 8) + b] - e.p(L.spos)[3 * (a & 255) + b]; break;
    case OB_SITE_MINUS_SITE: v = e.p(L.spos)[3 * (a >> 8) + b] - e.p(L.spos)[3 * (a & 255) + b]; break;
    case OB_BODY_MINUS_BODY: v = e.p(L.xpos)[3 * (a >> 8) + b] - e.p(L.xpos)[3 * (a & 255) + b]; break;
    case OB_REL_POS_LAG:
    case OB_REL_QUAT_LAG: {
      if (fresh || prev == nullptr) break;
      int ps = a & 4095, qs = a >> 12, comp = b & 255, site = (b >> 8) & 255, body = (b >> 16) & 255;
      R Re[9], Ro[9], qo[4] = {prev[qs + 3], prev[qs], prev[qs + 1], prev[qs + 2]};  // cached quaternion is (x, y, z, w)
      q2mat(Re, e.p(L.xquat) + 4 * body);
      if (op == OB_REL_POS_LAG) {
        R d[3] = {prev[ps] - e.p(L.spos)[3 * site], prev[ps + 1] - e.p(L.spos)[3 * site + 1], prev[ps + 2] - e.p(L.spos)[3 * site + 2]}, r[3];
        m3mulTv(r, Re, d);
        v = r[comp];
      } else {
        R rel[9], q[4];
        if (e.state().obs_mod != nullptr) {
          // with observable modifiers the cache may be corrupted, so not unit-length: normalise it as the reference's quat2mat does
          // (transform_utils.py: q *= sqrt(2 / n), the identity when n < 4 eps); a unit cache needs no such step
          const R n = qo[0] * qo[0] + qo[1] * qo[1] + qo[2] * qo[2] + qo[3] * qo[3];
          if (n < R(8.881784197001252e-16)) { qo[0] = 1; qo[1] = 0; qo[2] = 0; qo[3] = 0; }
          else { const R sc = R(1) / r_sqrt(n); for (int k = 0; k < 4; k++) qo[k] *= sc; }
        }
        q2mat(Ro, qo);
        for (int i = 0; i < 3; i++)
          for (int j = 0; j < 3; j++) rel[3 * i + j] = Re[i] * Ro[j] + Re[3 + i] * Ro[3 + j] + Re[6 + i] * Ro[6 + j];
        mat2quat_wpos(rel, q);
        v = q[(comp + 1) & 3];
      }
      break;
    }
    default: v = 0;
  }
  return v;
}

// Observable timers: Observable.update with delay 0 (utils/observables.py:214-259), called after every substep's step2
// (environments/base.py:494-505), one lane per observable, in fp64 in both precisions so the sample instants follow Python's floats:
//   t += dt;  if (force or (not sampled and t <= T)): sample, sampled = 1;  if (t >= T): (sample if not sampled), sampled = 0, t = fmod(t, T)
// Returns the mask of the observables that sample now.  `only_fresh` (forward()): only an environment whose observation cache is empty
// (just reset) samples, with reset()'s forced update (environments/base.py:418-427): t = 0, sampled = 0, then the update with force.
// Without modifiers (DState::obs_mod null) every observable samples on the last substep, which is where this rule puts the samples of
// the default rate.  The timers live out of line: inlined, their fp64 code (fmod) cost the tail's default path spill slots.
template <typename R> DEVN unsigned obs_timers(const Eng<R> e, int env, bool only_fresh) {
  const ObsModDev* om = e.state().obs_mod;
  if (only_fresh && !e.state().obs_fresh[env]) return 0u;
  const int n = om->nobs, lane = e.lane;
  const size_t i = (size_t)env * n + lane;
  bool sampled = !only_fresh && ((om->sampled[env] >> lane) & 1), due = false;
  if (lane < n) {
    const double T = om->period[lane];
    double t = __dadd_rn(only_fresh ? 0.0 : om->timer[i], om->dt);
    if (only_fresh || (!sampled && t <= T)) { due = true; sampled = true; }
    if (t >= T) {
      if (!sampled) due = true;
      sampled = false;
      t = fmod(t, T);
    }
    om->timer[i] = t;
  }
  const unsigned dm = __ballot_sync(B2S_FULL, due), sm = __ballot_sync(B2S_FULL, sampled && lane < n);
  if (lane == 0) om->sampled[env] = (int)sm;
  return dm;
}
template <typename R> DEV unsigned obs_due(const Eng<R>& e, int env, bool last, bool only_fresh) {
  return e.state().obs_mod == nullptr ? (last ? ~0u : 0u) : obs_timers(e, env, only_fresh);
}

// Corruptor of observation row k of a sample (create_gaussian_noise_corrupter / create_uniform_noise_corrupter, utils/observables.py):
// Philox4x32-10 keyed by the seed, counter (env, the observable's sample count, row, 0), so an environment's noise depends on neither the
// batch nor the mask.  u1, u2 = 53 bits of output words (0, 1) and (2, 3) as in perturb_kernel.
//   Gaussian  v + (mean + std * z),  z = sqrt(-2 log(1 - u1)) cos(2 pi u2)      Uniform  v + (min + (max - min) u1)
// then clipped to [low, high], in fp64 without contraction, rounded to the handle's precision last.
template <typename R> DEV R obs_corrupt(const ObsModDev* om, int env, int k, R v) {
  const int o = om->row_obs[k], kind = om->kind[o];
  if (kind == OBS_CORRUPT_NONE) return v;
  const unsigned cnt = (unsigned)om->nsample[(size_t)env * om->nobs + o];
  const uint4 x = philox4x32_10(make_uint4((unsigned)env, cnt, (unsigned)k, 0u), (unsigned)om->seed, (unsigned)(om->seed >> 32));
  const double u1 = (double)(((unsigned long long)(x.x >> 5) << 26) | (x.y >> 6)) * 0x1p-53;
  double d;
  if (kind == OBS_CORRUPT_GAUSSIAN) {
    const double u2 = (double)(((unsigned long long)(x.z >> 5) << 26) | (x.w >> 6)) * 0x1p-53;
    const double z = __dmul_rn(sqrt(__dmul_rn(-2.0, log(__dsub_rn(1.0, u1)))), cos(__dmul_rn(6.283185307179586, u2)));
    d = __dadd_rn(om->p0[o], __dmul_rn(om->p1[o], z));
  } else {
    d = __dadd_rn(om->p0[o], __dmul_rn(__dsub_rn(om->p1[o], om->p0[o]), u1));
  }
  return (R)fmin(fmax(__dadd_rn((double)v, d), om->lo[o]), om->hi[o]);
}

// The observation rows of the observables in `due` (bit o: observable o = obs_mod->row_obs[row]; without modifiers every row).
// `only_fresh`: called from forward() - sample only environments whose observation cache is empty (just reset)
template <typename R> DEVN void write_obs(const Eng<R> e, int env, bool only_fresh, unsigned due) {
  const DState<R>& s = e.state();
  const CtrlCfgDev& cc = e.ccfg();
  const ObsModDev* om = s.obs_mod;
  R* out = s.obs + (size_t)env * cc.obs_dim;
  int fresh = s.obs_fresh[env];
  if (only_fresh && !fresh) return;
  R val[4];  // obs_dim <= 128: all values are formed before any is written (lagged entries read the previous sample)
  unsigned on = 0;
#pragma unroll 1
  for (int it = 0; it < 4; it++) {  // rolled: table_value is large and runs once per sample
    int k = e.lane + 32 * it;
    const bool take = k < cc.obs_dim && (om == nullptr || ((due >> om->row_obs[k]) & 1));
    val[it] = take ? table_value(e, cc.obs_op[k], cc.obs_a[k], cc.obs_b[k], out, fresh) : R(0);
    if (take && om) val[it] = obs_corrupt(om, env, k, val[it]);
    on |= (unsigned)take << it;
  }
  __syncwarp();
#pragma unroll 1
  for (int it = 0; it < 4; it++) {
    int k = e.lane + 32 * it;
    if ((on >> it) & 1) out[k] = val[it];
  }
  if (e.lane == 0 && fresh) s.obs_fresh[env] = 0;
  if (om && e.lane < om->nobs && ((due >> e.lane) & 1)) om->nsample[(size_t)env * om->nobs + e.lane]++;
}

// Task outputs after the last substep (poses / contacts of the last step1, as the reference's reward() sees them:
// manipulation/lift.py:224-273,433-444; manipulation_env.py:331-376 _check_grasp; utils/sim_utils.py:8-40)
template <typename R> DEVN void write_task(const Eng<R> e, int env, int ncon) {
  const DModel<R>& m = e.model();
  const WSLayout& L = e.lay();
  const DState<R>& s = e.state();
  const CtrlCfgDev& cc = e.ccfg();
  const int* cint = e.pi(L.c_int);
  int hitl = 0, hitr = 0, hit2 = 0, hl4 = 0, hr4 = 0;
  for (int c = e.lane; c < ncon; c += 32) {
    unsigned long long b1 = 1ull << m.geom_cgid[cint[5 * c]], b2 = 1ull << m.geom_cgid[cint[5 * c + 1]];
    for (int i = 0; i < cc.n_objs; i++) {
      bool p1 = b1 & cc.mask_objs[i], p2 = b2 & cc.mask_objs[i];
      if ((p1 && (b2 & cc.mask_left)) || (p2 && (b1 & cc.mask_left))) hl4 |= 1 << i;
      if ((p1 && (b2 & cc.mask_right)) || (p2 && (b1 & cc.mask_right))) hr4 |= 1 << i;
    }
    bool o1 = b1 & cc.mask_obj, o2 = b2 & cc.mask_obj;
    if ((o1 && (b2 & cc.mask_left)) || (o2 && (b1 & cc.mask_left))) hitl = 1;
    if ((o1 && (b2 & cc.mask_right)) || (o2 && (b1 & cc.mask_right))) hitr = 1;
    if ((o1 && (b2 & cc.mask_obj2)) || (o2 && (b1 & cc.mask_obj2))) hit2 = 1;
  }
  hitl = warp_or_i(hitl); hitr = warp_or_i(hitr); hit2 = warp_or_i(hit2);
  if (cc.n_objs > 0) { hl4 = warp_or_i(hl4); hr4 = warp_or_i(hr4); }
  if (e.lane == 0) {
    R* out = s.task_out + (size_t)env * 8;
    const R* bp = e.p(L.xpos) + 3 * cc.task_body; const R* sp = e.p(L.spos) + 3 * cc.task_site;
    R d[3];
    v3sub(d, bp, sp);
    out[0] = bp[2]; out[1] = v3norm(d); out[2] = (hitl && hitr) ? R(1) : R(0);
    R hd = 0;
    if (cc.task_body2 >= 0) { const R* b2p = e.p(L.xpos) + 3 * cc.task_body2; hd = r_sqrt((bp[0] - b2p[0]) * (bp[0] - b2p[0]) + (bp[1] - b2p[1]) * (bp[1] - b2p[1])); }
    out[3] = hd; out[4] = hit2 ? R(1) : R(0); out[5] = (R)(hl4 & hr4); out[6] = 0; out[7] = 0;
  }
  // task table: poses the task's reward / success checks read after the step (same scalar ops as the observation table)
  for (int k = e.lane; k < cc.task_dim; k += 32)
    s.task_vec[(size_t)env * cc.task_dim + k] = table_value(e, cc.task_op[k], cc.task_a[k], cc.task_b[k], (const R*)nullptr, 0);
  __syncwarp();  // orders warn bit 512 of a selection op (any lane) before store_state's read-modify-write (lane 0)
}

// controller.reset_goal + initial joints (osc.py:520-544, controller.py:126-132): goal <- current eef pose (world),
// initial_joint <- current arm qpos, gripper integrator <- 0.  Uses the exported site arrays of a prior forward.
template <typename R>
__global__ void ctrl_reset_kernel(const uint8_t* mask, int slot) {
  const DModel<R>& m = cmodel<R>(slot);
  const DState<R>& s = cstate<R>(slot);
  const CtrlCfgDev& cc = c_cc[slot];
  int env = blockIdx.x * blockDim.x + threadIdx.x;
  if (env >= s.n_env) return;
  if (mask && !mask[env]) return;
  size_t E = env;
  for (int k = 0; k < 3; k++) s.goal_pos[E * 3 + k] = s.site_xpos[(E * m.nsite + cc.eef_site) * 3 + k];
  for (int k = 0; k < 9; k++) s.goal_ori[E * 9 + k] = s.site_xmat[(E * m.nsite + cc.eef_site) * 9 + k];
  for (int k = 0; k < cc.n_arm; k++) s.init_qpos_arm[E * 8 + k] = s.qpos[E * m.nq + cc.arm_qpos[k]];
  for (int k = 0; k < 4; k++) s.grip_state[E * 4 + k] = 0;
  for (int k = 0; k < 72; k++) s.jv_state[E * 72 + k] = k == 64 ? R(4) : R(0);  // ring pointer starts at length - 1
  if (cc.kind == 3)  // JointPositionController.reset_goal: goal <- current joint positions
    for (int k = 0; k < cc.n_arm; k++) s.jv_state[E * 72 + k] = s.qpos[E * m.nq + cc.arm_qpos[k]];
  if (cc.gain)  // variable impedance: the rebuilt controller starts from the configured gains
    for (int k = 0; k < 8; k++) {
      const bool osc = cc.kind != 3, on = k < (osc ? 6 : cc.n_arm);
      cc.gain[E * 16 + k] = on ? (osc ? cc.kp[k] : cc.jv_kp[k]) : 0.0;
      cc.gain[E * 16 + 8 + k] = on ? (osc ? cc.kd[k] : cc.jv_kd[k]) : 0.0;
    }
}
