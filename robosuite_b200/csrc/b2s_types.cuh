// Device-side model / workspace descriptors of the batched engine (one environment per warp).
// The field set mirrors what the reference reads from the engine through binding_utils.MjModel / MjData
// (robosuite/utils/binding_utils.py:252-1056); layouts are this repo's own.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define B2S_FULL 0xffffffffu
#define B2S_MOV 8  // per-handle cap of b2s_model_override: geoms, and separately bodies

enum { JNT_FREE = 0, JNT_BALL = 1, JNT_SLIDE = 2, JNT_HINGE = 3 };
enum { G_PLANE = 0, G_HFIELD, G_SPHERE, G_CAPSULE, G_ELLIPSOID, G_CYLINDER, G_BOX, G_MESH };
enum { C_FRICTION = 1, C_LIMIT = 3, C_FRICTIONLESS = 5, C_ELLIPTIC = 7 };
// dof kinds (precomputed on the host): how cdof is formed from the owning body's pose
enum { DK_FREE_T = 0, DK_FREE_R = 1, DK_SLIDE = 2, DK_HINGE = 3 };

// kernel phase flags
enum {
  PH_STEP1 = 1,      // position + velocity stage
  PH_STEP2 = 2,      // actuation, solve, integrate
  PH_NOINTEGRATE = 4,  // forward(): everything of step2 except the Euler update
  PH_EXPORT = 8,     // write derived arrays (xpos, qM, contacts, efc ...) to HBM
  PH_CTRL = 16,      // run the fused controller between step1 and step2
  PH_CTRL_EXT = 512, // pipeline mode: the controller ran as its own kernel (ctrl_osc_kernel), `ctrl` is already in HBM
  PH_OBS = 64        // write the observation row and the task outputs (after the last substep)
};

template <typename R>
struct DModel {
  int nq, nv, nu, nbody, njnt, ngeom, nsite, npair, ncg, nment, maxdepth, maxcon, maxefc, nmocap, nfl, nlim, nspr, hc_stride, max_treesize;
  int stage_cap;  // reals of shared memory the convex narrow-phase kernel has for staging the hull vertices of a pair
  R timestep, impratio, density, viscosity, tolerance, meaninertia;
  int iterations, ls_iterations;
  R gravity[3], wind[3];
  // bodies
  const int *body_parentid, *body_jntid, *body_dofnum, *body_dofadr, *body_weldid, *body_subtree_end, *body_depth;
  const R *body_pos, *body_quat, *body_ipos, *body_iquat, *body_mass, *body_inertia, *body_invweight0;
  const R *body_xpos0, *body_xquat0;  // world pose of bodies welded to the world (constant)
  // joints
  const int *jnt_type, *jnt_qposadr, *jnt_dofadr, *jnt_bodyid, *jnt_limited;
  const R *jnt_pos, *jnt_axis, *jnt_range, *jnt_margin, *jnt_solref, *jnt_solimp, *qpos0;
  const int* spr_jnt;                       // the nspr hinge and slide joints with nonzero stiffness
  const R *jnt_stiffness, *qpos_spring;     // spring force -stiffness (qpos - qpos_spring) on the listed joints
  // dofs
  const int *dof_bodyid, *dof_jntid, *dof_parentid, *dof_kind, *dof_cddstart, *fl_dof, *lim_jnt, *dof_treebase, *dof_treesize, *body_treeid;
  const unsigned long long* body_dofmask;  // bit i set: dof i is on the chain of this body
  const R *dof_armature, *dof_damping, *dof_frictionloss, *dof_solref, *dof_solimp, *dof_invweight0;
  // nonzero lower-triangular mass-matrix entries (i >= j, j on the chain of i)
  const int *ment_i, *ment_j;
  // geoms
  const int *geom_type, *geom_bodyid, *geom_condim, *geom_dataid, *geom_priority, *geom_cgid, *cg_geom;
  const R *geom_size, *geom_pos, *geom_quat, *geom_friction, *geom_solmix, *geom_solref, *geom_solimp, *geom_rbound,
      *geom_aabb;
  const int* pair_geom;
  const int *mesh_vertadr, *mesh_vertnum;
  const R* mesh_vert;
  // sites
  const int* site_bodyid;
  const R *site_pos, *site_quat;
  // actuators
  const int *act_trnid, *act_ctrllimited, *act_forcelimited, *act_biastype;
  const R *act_ctrlrange, *act_forcerange, *act_gear, *act_gainprm, *act_biasprm;
};

// Per-environment arrays in HBM (row-major [n_env][k]: a warp reads its environment's row coalesced).
template <typename R>
struct DState {
  int n_env;
  R *qpos, *qvel, *qacc, *qacc_ws, *ctrl, *time;
  // exported derived arrays (PH_EXPORT)
  R *xpos, *xquat, *xmat, *site_xpos, *site_xmat, *geom_xpos, *geom_xmat, *qM, *qfrc_bias, *qfrc_passive,
      *qfrc_actuator, *qfrc_constraint, *qfrc_smooth, *qacc_smooth, *actuator_force, *cdof;
  int *ncon, *contact_geom, *contact_dim, *nefc, *efc_type, *warn, *solver_niter;
  R *contact_dist, *contact_pos, *contact_frame, *contact_friction, *contact_solref, *contact_solimp, *efc_J, *efc_force,
      *efc_aref, *efc_D, *efc_R;
  // fused controller state / io
  R *goal_pos, *goal_ori, *init_qpos_arm, *grip_state;
  R* ctrl_torque;  // exported arm torques before clipping (tests)
  R* jv_state;     // [n_env, 72] JOINT_VELOCITY: goal 8, last_err 8, summed 8, derr ring 5x8, ptr, size, saturated
  R* obs;          // [n_env, obs_dim] sampled after the first substep of a control step (observables.py:230-240)
  R* wsg;          // [n_env, L.total] global workspace rows (pipeline mode)
  // pipeline-mode collision work lists (candidate pairs of ALL environments, compacted with atomics)
  int* cl_cnt;     // per group [CL_CNT_STRIDE]: number of analytic / convex candidates this substep, (spare), next convex work item,
                   // (spare x4), then environments per tail cost class for even / odd substeps [2][TAIL_NKEY]
  int cl_maxa, cl_maxg;  // per-environment candidate capacity of the two work lists
  int* cl_listA;   // [n_env * cl_maxa] env << 12 | pair
  int* cl_listG;   // [n_env * cl_maxg]
  R* cl_outA;      // [n_env * cl_maxa][CL_RECA] count + 8 x (pos3 normal3 dist)
  R* cl_outG;      // [n_env * cl_maxg][8]       count + (pos3 normal3 dist)
  R* gjk_cache;    // [n_env][npair][3] last separating direction of each convex pair (GJK warm start)
  int* cl_env;     // [n_env][2 + 2 * (cl_maxa + cl_maxg)] na, ng, then (pair, slot) of each candidate
  // pipeline-mode tail order: a group's tail launch runs its environments most expensive cost class first when tail_sorted (a block
  // shape choice, choose_blocks), else by id
  int tail_sorted;
  int* tail_key;  // [n_env] cost class of the environment's last tail (tail_cost_key)
  int* tail_list;  // [n_env * TAIL_NKEY] per group (from env0 * TAIL_NKEY) and class k (at + k * nenv): the environments phase 0 filed
  int* tail_order; // [n_env] per group: the environment the last tail launch ran at warp position p, at env0 + p
  int* obs_fresh;  // [n_env] 1 = observation cache empty (set at reset, cleared by the first sample)
  // per-environment world poses of bodies welded to the world (the reference writes sampled placements into model.body_pos /
  // body_quat per reset, e.g. the Door: door.py:417-427; model constants are shared by a batch here, so these are DATA): up to 4 bodies
  int n_ov, ov_body[4];
  R* ov_pos[4];    // [n_env, 3]
  R* ov_quat[4];   // [n_env, 4]
  // per-environment model values (b2s_model_override): up to B2S_MOV colliding primitive geoms (size, friction) and B2S_MOV moving
  // bodies (mass, principal moments).  Slot k of environment e sits at [k * n_env + e].  n_mg == n_mb == 0 and null derived
  // arrays: the handle has no overrides and every lookup (b2s_engine.cuh, *_of) costs one warp-uniform test.
  int n_mg, n_mb;
  short mg_id[B2S_MOV], mb_id[B2S_MOV];
  R *mg_size, *mg_fric, *mg_rbound, *mg_aabb;  // [B2S_MOV][n_env] x 3 / 3 / 1 / 6 (rbound, aabb: written by the set-constants pass)
  R *mb_mass, *mb_inertia;                     // [B2S_MOV][n_env] x 1 / 3
  R *mg_solref, *mg_solimp;                    // [B2S_MOV][n_env] x 2 / 5 (same geom slots as size and friction)
  R *dof_iw, *body_iw, *mean_inertia;          // [n_env] x nv / nbody * 2 / 1: dof_invweight0, body_invweight0, meaninertia
  // whole-vector dof overrides, [n_env, nv] each; null = the model's vector.  A non-null dof_floss makes the friction-loss rows
  // per environment (the dofs whose own value is > 0) instead of the model's static list
  R *dof_damp, *dof_arm, *dof_floss;
  R* task_vec;     // [n_env, task_dim] task table values after the last substep
  R* task_out;     // [n_env, 8]: body height, |grip site - body|, grasp flag, horizontal |body - body2|, obj-obj2 contact flag
  // -DB2S_INSTR builds only (measurement aid, see b2s_instr in b2s_pipeline.cuh): device timeline of the graph replay and
  // solver statistics.  Null in product builds.
  unsigned long long* st_begin;  // [64 groups][32 substeps][8 kernel kinds] first %globaltimer of the launch
  unsigned long long* st_end;    //                                     last %globaltimer of the launch
  int* stats;      // [512]: 0..15 Newton-iteration histogram, 16 line-search evaluations, 17 solves, 19 large-tier environments,
                   // 32..160 ncon histogram, 176..496 nefc histogram
  float* cyc;      // [n_env][32 substeps][8] per environment-substep: clock64 cycles of its warp in P0, in the tail kernel; then the
                   // tail's Newton iterations, line-search evaluations, nefc, ncon, capacity tier (1 = large) and tail block index
  int* solve_ls;   // [n_env] line-search evaluations of the environment's last Newton solve
  int* slowlog;    // [64][12] convex work items above 131 k cycles: cycles, shape types, hull sizes, EPA nV nF, GJK cycles, hit, staged, geoms
  const struct ObsModDev* obs_mod;  // sampling rates and corruptors (b2s_obs_modifiers); null: every observable on the last substep, no noise
};

// offsets (in units of R) of the per-warp shared-memory workspace
struct WSLayout {
  int qpos, qvel, qacc, qacc_ws, ctrl;
  int xpos, xquat, xmat, xipos;
  int cdof, cdofdot, cinert, cvel, frne, ffl;
  int M, H;
  int bias, passive, qact, qsmooth, qaccs, qcon;
  int gpos, gmat, spos, smat;
  int c_pos, c_frame, c_dist, c_fric, c_solref, c_solimp, c_mu, c_int;  // c_int: 5 ints per contact (g1,g2,dim,adr,pair)
  int J, e_D, e_R, e_aref, e_jar, e_jv, e_force, e_floss, e_int;        // e_int: 2 ints per row (type,id)
  int Ma, grad, search, Mv;
  int scratch, scratch_size;
  int fused_stride;  // words per warp in the fused kernel = total + EPA polytope area
  int hdr;  // 8 words of per-env integers passed between pipeline phases: ncon, nefc, warn, niter
  int total;
  int mc, me;  // contact / constraint-row capacity of THIS layout (the small tier of the tail kernel holds fewer than the model's
               // maxcon / maxefc; environments that need more are re-run with the large tier)
};

// A handle owns one slot of every descriptor array below; a kernel is told its slot and which of the slot's layouts its warps use:
// the full layout (fused kernel), phase 0's, the tail kernel's small / large tier, and the layout of the global workspace row.
#define B2S_NSLOT 8
enum { LAY_FULL = 0, LAY_P0 = 1, LAY_TS = 2, LAY_TL = 3, LAY_ROW = 4, B2S_NLAY = 5 };

// Pipeline mode: the substep is split into phase kernels; each phase loads / stores these workspace regions
// from / to the per-environment global workspace row (L2 resident).
struct Region { int off, goff, len, dyn; };  // shared-memory offset, offset in the global row, words; dyn: 1 = nefc*nv words
// PhaseIO slots: what phase 0 stores, what the tail kernel loads at its start / before the observation sample, per tier
enum { PIO_P0 = 0, PIO_TS = 1, PIO_TS_LATE = 2, PIO_TL = 3, PIO_TL_LATE = 4, B2S_NPIO = 5 };
#define CL_MAXA 64  // hard upper bounds of the per-environment candidate counts (analytic / convex pairs);
#define CL_MAXG 32  // the run-time caps DState::cl_maxa / cl_maxg are chosen per model (b2s_capi.cu)
#define CL_RECA 58
#define CL_ENVW(s) (2 + 2 * ((s).cl_maxa + (s).cl_maxg))
#define TAIL_NKEY 16                          // tail cost classes (tail_cost_key, b2s_pipeline.cuh)
#define TAIL_SOLO 2                           // tail blocks whose one expensive environment runs beside cheap ones (tail_env_at)
#define CL_CNT_STRIDE (8 + 2 * TAIL_NKEY)     // ints per group in DState::cl_cnt
#define B2S_MAXREG 12
// load / store lists hold merged 16-byte aligned spans; load_words = sum of the fixed spans, load_dyn = list has the Jacobian
struct PhaseIO { int nload, nstore, load_words, load_dyn; Region load[B2S_MAXREG], store[B2S_MAXREG]; };

// observation scalar ops (one table entry per output scalar)
enum { OB_QPOS = 0, OB_COS_QPOS, OB_SIN_QPOS, OB_QVEL, OB_QACC, OB_SITE_POS, OB_BODY_POS, OB_BODY_QUAT_XYZW, OB_SITE_QUAT_XYZW,
       OB_BODY_MINUS_SITE, OB_SITE_MINUS_SITE, OB_BODY_QUAT_REL_SITE_XYZW, OB_ZERO, OB_BODY_MINUS_BODY,
       // object pose in the gripper frame from the object pose of the PREVIOUS observation sample (the reference evaluates
       // `{obj}_to_eef_pos/quat` before `{obj}_pos/quat` in the same pass: manipulation_env.py:268-329) and the current
       // hand pose; zeros on the first sample after a reset.  a = pos_slot | quat_slot << 12, b = k | site << 8 | body << 16
       OB_REL_POS_LAG, OB_REL_QUAT_LAG };

// Observable sampling rates and corruptors (b2s_obs_modifiers), kept in device memory (the constant bank is nearly full).  Per
// observable o: period T = 1 / sampling_rate and the corruptor (kind: B2S_CORRUPT_* of include/b2s.h; p0, p1 = mean, std or
// min_noise, max_noise; clip range [lo, hi]).  Per environment: the time since the last period boundary, the flags of the
// observables sampled in the current period, and the samples each observable took (the noise counter, never rewound).
#define B2S_MAXOBS 32
struct ObsModDev {
  int nobs;
  unsigned long long seed;
  double dt;  // the model's timestep in fp64 in both precisions: the reference's timers are Python floats
  double period[B2S_MAXOBS], p0[B2S_MAXOBS], p1[B2S_MAXOBS], lo[B2S_MAXOBS], hi[B2S_MAXOBS];
  int kind[B2S_MAXOBS];
  int row_obs[128];  // the observable of each observation row
  double* timer;     // [n_env, nobs]
  int* sampled;      // [n_env] bit o: observable o has sampled in its current period
  int* nsample;      // [n_env, nobs]
};
enum { OBS_CORRUPT_NONE = 0, OBS_CORRUPT_GAUSSIAN = 1, OBS_CORRUPT_UNIFORM = 2 };  // = B2S_CORRUPT_* (include/b2s.h)

struct CtrlCfgDev {
  int kind, action_dim, n_arm, eef_site, base_site, n_grip, uncouple;
  int obs_dim; const int* obs_op; const int* obs_a; const int* obs_b;  // device arrays
  int task_body, task_site; unsigned long long mask_left, mask_right, mask_obj;  // grasp check geom sets (colliding-geom index bits)
  int task_body2; unsigned long long mask_obj2;  // second object (Stack: cubeB), -1 / 0 when unused
  int n_objs; unsigned long long mask_objs[4];   // per-object grasp flags (multi-object tasks)
  int task_dim; const int* task_op; const int* task_a; const int* task_b;  // task table (device arrays)
  // JOINT_VELOCITY part controller (controllers/parts/generic/joint_vel.py)
  double jv_kp[8], jv_ki[8], jv_kd[8], jv_in_max[8], jv_in_min[8], jv_out_max[8], jv_out_min[8], jv_vel_lo, jv_vel_hi;
  int jv_use_vel_limits, jv_torque_comp;
  int arm_dof[8], arm_qpos[8], arm_act[8], grip_act[4];
  double grip_sign[4], grip_speed, kp[6], kd[6], input_max[6], input_min[6], output_max[6], output_min[6], null_kp;
};

// ---- constant-memory descriptors, one slot per live handle (b2s_create takes a free slot, b2s_destroy returns it).  Device code
// reads them through the constant bank with a warp-uniform slot index, so non-inlined phase functions need no descriptor
// arguments beyond the (slot, layout) pair carried by Eng, and handles of different tasks run concurrently on one GPU.
__constant__ DModel<float> c_model_f[B2S_NSLOT];
__constant__ DModel<double> c_model_d[B2S_NSLOT];
__constant__ DState<float> c_state_f[B2S_NSLOT];
__constant__ DState<double> c_state_d[B2S_NSLOT];
__constant__ WSLayout c_lay[B2S_NSLOT][B2S_NLAY];
__constant__ CtrlCfgDev c_cc[B2S_NSLOT];
__constant__ PhaseIO c_pio[B2S_NSLOT][B2S_NPIO];
template <typename R> __device__ __forceinline__ const DModel<R>& cmodel(int slot);
template <> __device__ __forceinline__ const DModel<float>& cmodel<float>(int slot) { return c_model_f[slot]; }
template <> __device__ __forceinline__ const DModel<double>& cmodel<double>(int slot) { return c_model_d[slot]; }
template <typename R> __device__ __forceinline__ const DState<R>& cstate(int slot);
template <> __device__ __forceinline__ const DState<float>& cstate<float>(int slot) { return c_state_f[slot]; }
template <> __device__ __forceinline__ const DState<double>& cstate<double>(int slot) { return c_state_d[slot]; }
