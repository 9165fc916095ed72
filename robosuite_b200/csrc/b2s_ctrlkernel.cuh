// Operational-space controller outside the per-warp tail kernel: ONE THREAD per environment.
//
// Inside the per-warp tail kernel the controller was 25 % of the time: serial 7x7 / 6x6 fp64 algebra on <= 8 of 32 lanes, ~4100 warp
// instructions per environment-substep.  The same arithmetic with one environment per LANE keeps all 32 lanes busy (~90 warp
// instructions per environment-substep), has no divergence (the controller is branch-free except for the singular-pose path) and
// depends only on phase 0's outputs (site poses, motion axes, M, bias, body velocities), so it runs beside the collision narrow
// phase: as one of the three block roles of the phase-1 kernel (b2s_pipeline.cuh).  Work arrays are columns of a shared-memory tile ([k][lane]: conflict-free), the arithmetic is b2s_oscmath.h - the very
// source the host test compiles and checks against the oracle / the reference's OperationalSpaceController.
// Reference: OperationalSpaceController.set_goal / run_controller (controllers/parts/arm/osc.py:225-283, 403-495),
// SimpleGripController (parts/gripper/simple_grip.py:150-186), FixedBaseRobot.control clipping (robots/fixed_base_robot.py:149-153).
#pragma once
#include "b2s_ctrl.cuh"
#include "b2s_oscmath.h"

#define OSC_TPB 32
template <typename R> constexpr size_t osc_smem_bytes() { return (size_t)OSC_TPB * (OSC_WORK_DOUBLES * sizeof(double) + 6 * OSC_NA_MAX * sizeof(R)); }

// body of one 32-thread block (role block `rb` of the phase-1 kernel, b2s_pipeline.cuh): environments rb * 32 .. rb * 32 + 31 of the group
template <typename R>
DEV void ctrl_osc_block(int sub, const R* action, int env0, int nenv, int gid, int slot, unsigned char* smem_raw, int rb) {
  const DModel<R>& m = cmodel<R>(slot);
  const DState<R>& s = cstate<R>(slot);
  const WSLayout& L = c_lay[slot][LAY_ROW];  // inputs come from phase 0's global workspace row
  const CtrlCfgDev& cc = c_cc[slot];
  double* wd = reinterpret_cast<double*>(smem_raw);                          // [OSC_WORK_DOUBLES][OSC_TPB]
  R* jt = reinterpret_cast<R*>(wd + (size_t)OSC_WORK_DOUBLES * OSC_TPB);      // [6 * OSC_NA_MAX][OSC_TPB]
  const int t = threadIdx.x, idx = rb * OSC_TPB + t;
  if (idx >= nenv) return;
  const int env = env0 + idx, na = cc.n_arm, nv = m.nv;
  const size_t E = env;
  const R* row = s.wsg + E * L.total;
  const R* ref_pos = row + L.spos + 3 * cc.eef_site; const R* ref_ori = row + L.smat + 9 * cc.eef_site;
  const R* org_pos = row + L.spos + 3 * cc.base_site; const R* org_ori = row + L.smat + 9 * cc.base_site;
  R rp[3], ro[9], op[3], oo[9];
#pragma unroll
  for (int k = 0; k < 3; k++) { rp[k] = ref_pos[k]; op[k] = org_pos[k]; }
#pragma unroll
  for (int k = 0; k < 9; k++) { ro[k] = ref_ori[k]; oo[k] = org_ori[k]; }
  R goal_pos[3], goal_ori[9], grip[4];
#pragma unroll
  for (int k = 0; k < 3; k++) goal_pos[k] = s.goal_pos[E * 3 + k];
#pragma unroll
  for (int k = 0; k < 9; k++) goal_ori[k] = s.goal_ori[E * 9 + k];
#pragma unroll
  for (int k = 0; k < 4; k++) grip[k] = s.grip_state[E * 4 + k];
  if (sub == 0 && action != nullptr) {  // policy step: set_goal (osc.py:225-283) + gripper format_action
    const R* act = action + E * cc.action_dim;
    if (cc.gain) {  // variable impedance: the gains first, then the delta that follows them
      for (int k = 0; k < 6; k++) imp_gain(cc.imp, act, k, cc.gain + E * 16 + k, cc.gain + E * 16 + 8 + k);
      act += cc.imp->off;
    }
    const int od = cc.kind == 5 ? 3 : 6;  // OSC_POSITION: no orientation delta, goal_ori re-anchored to the current orientation
    R sd[6] = {0, 0, 0, 0, 0, 0};
    for (int k = 0; k < od; k++) {
      R a = r_clamp(act[k], (R)cc.input_min[k], (R)cc.input_max[k]);
      R scale = (R)(fabs(cc.output_max[k] - cc.output_min[k]) / fabs(cc.input_max[k] - cc.input_min[k]));
      sd[k] = (a - (R)(0.5 * (cc.input_max[k] + cc.input_min[k]))) * scale + (R)(0.5 * (cc.output_max[k] + cc.output_min[k]));
    }
    R rel[3], inb[3], cur[9], Rd[9];
    v3sub(rel, rp, op);
    m3mulTv(inb, oo, rel);
    for (int k = 0; k < 3; k++) goal_pos[k] = inb[k] + sd[k];
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) cur[3 * i + j] = oo[i] * ro[j] + oo[3 + i] * ro[3 + j] + oo[6 + i] * ro[6 + j];
    delta_rotmat(Rd, sd + 3);
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) goal_ori[3 * i + j] = Rd[3 * i] * cur[j] + Rd[3 * i + 1] * cur[3 + j] + Rd[3 * i + 2] * cur[6 + j];
    R ga = act[od];
    R sg = ga > 0 ? R(1) : (ga < 0 ? R(-1) : R(0));
    for (int gI = 0; gI < cc.n_grip; gI++) grip[gI] = r_clamp(grip[gI] + (R)(cc.grip_sign[gI] * cc.grip_speed) * sg, R(-1), R(1));
    for (int k = 0; k < 3; k++) s.goal_pos[E * 3 + k] = goal_pos[k];
    for (int k = 0; k < 9; k++) s.goal_ori[E * 9 + k] = goal_ori[k];
    for (int k = 0; k < 4; k++) s.grip_state[E * 4 + k] = grip[k];
  }
  // ---- gather this environment's inputs from phase 0's workspace row
  OscView<R> J{jt + t, OSC_TPB};
  OscView<double> W{wd + t, OSC_TPB};
  const int eb = m.site_bodyid[cc.eef_site], bb = m.site_bodyid[cc.base_site];
  const unsigned long long emask = m.body_dofmask[eb];
  const R* cdof = row + L.cdof; const R* M = row + L.M;
  for (int a = 0; a < na; a++) {
    int i = cc.arm_dof[a];
    R col[6] = {0, 0, 0, 0, 0, 0};
    if ((emask >> i) & 1ull) {
      R cd[6];
#pragma unroll
      for (int k = 0; k < 6; k++) cd[k] = cdof[6 * i + k];
      osc_jac_col(cd, rp, col);
    }
#pragma unroll
    for (int r = 0; r < 6; r++) J[r * na + a] = col[r];
    for (int b = 0; b <= a; b++) W[OSC_OFF_L + osc_tri(a, b)] = (double)M[i * nv + cc.arm_dof[b]];
  }
  R cve[6], cvb[6], vel[6], bvel[6];
#pragma unroll
  for (int k = 0; k < 6; k++) { cve[k] = row[L.cvel + 6 * eb + k]; cvb[k] = row[L.cvel + 6 * bb + k]; }
  osc_jac_col(cve, rp, vel);   // site velocity [linear; angular] from the owning body's spatial velocity
  osc_jac_col(cvb, op, bvel);
  double F[6], pt[OSC_NA_MAX], bias[OSC_NA_MAX], tau[OSC_NA_MAX];
  if (cc.gain) osc_wrench(rp, ro, op, oo, goal_pos, goal_ori, vel, bvel, cc.gain + E * 16, cc.gain + E * 16 + 8, F);
  else osc_wrench(rp, ro, op, oo, goal_pos, goal_ori, vel, bvel, cc.kp, cc.kd, F);
  const double kv = 2.0 * sqrt(cc.null_kp);
#pragma unroll
  for (int a = 0; a < OSC_NA_MAX; a++) {
    if (a < na) {
      int i = cc.arm_dof[a];
      pt[a] = cc.null_kp * ((double)s.init_qpos_arm[E * 8 + a] - (double)s.qpos[E * m.nq + cc.arm_qpos[a]]) - kv * (double)s.qvel[E * nv + i];
      bias[a] = (double)row[L.bias + i];
    } else { pt[a] = 0; bias[a] = 0; }
  }
  osc_torques(J, W, na, F, pt, bias, cc.uncouple, tau);
  // ---- FixedBaseRobot.control: clip to the actuator ctrlrange, write ctrl
  R* ctrl = s.ctrl + E * m.nu;
#pragma unroll
  for (int a = 0; a < OSC_NA_MAX; a++) {
    if (a < na) {
      int u = cc.arm_act[a];
      s.ctrl_torque[E * 8 + a] = (R)tau[a];
      ctrl[u] = r_clamp((R)tau[a], m.act_ctrlrange[2 * u], m.act_ctrlrange[2 * u + 1]);
    }
  }
  for (int gI = 0; gI < cc.n_grip; gI++) {
    int u = cc.grip_act[gI];
    R lo = m.act_ctrlrange[2 * u], hi = m.act_ctrlrange[2 * u + 1];
    ctrl[u] = r_clamp(R(0.5) * (hi + lo) + R(0.5) * (hi - lo) * grip[gI], lo, hi);
  }
  (void)gid;
}
