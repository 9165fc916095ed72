/* libb2s - C ABI of the H100-native batched rigid-body engine (one environment per warp, sm_90a).
 *
 * Every entry point replaces one call the reference makes into its third-party engine through
 * `robosuite/utils/binding_utils.py` (the `MjSim` shim, SURVEY.md section 8b "Seam 1"), batched over n_env
 * independent environments.  All array arguments are DEVICE pointers unless the name ends in `_host`.
 * Return value: 0 on success, negative error code otherwise; `b2s_last_error()` returns a thread-local message
 * (the Python layer maps codes to the exception types of `robosuite/utils/errors.py`).
 * A handle is not thread-safe (matches the reference: one MjSim per env per process, binding_utils.py:1059).
 */
#ifndef B2S_H
#define B2S_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b2s_sim b2s_sim;

enum { B2S_OK = 0, B2S_ERR_ARG = -1, B2S_ERR_CUDA = -2, B2S_ERR_MODEL = -3, B2S_ERR_UNSUPPORTED = -4 };
enum { B2S_F32 = 0, B2S_F64 = 1, B2S_I32 = 2, B2S_I64 = 3 };
/* controller kinds for the fused control step (controller_config "type", controllers/parts/controller_factory.py:145) */
/* arm part controllers: controllers/parts/arm/osc.py, parts/generic/joint_vel.py, joint_pos.py, joint_tor.py.  The two joint-space
 * kinds 3 / 4 keep their per-joint scaling in jv_in/out_*, their gains in jv_kp / jv_kd (kd = 2 sqrt(kp) damping_ratio). */
enum { B2S_CTRL_NONE = 0, B2S_CTRL_OSC_POSE = 1, B2S_CTRL_JOINT_VELOCITY = 2, B2S_CTRL_JOINT_POSITION = 3, B2S_CTRL_JOINT_TORQUE = 4,
       B2S_CTRL_OSC_POSITION = 5 /* controllers/parts/arm/osc.py:152-166: 3-dim arm action, orientation held */ };

/* MjSim.from_xml_string (binding_utils.py:1074-1087): `model_blob` is the flat compiled model produced by
 * robosuite_b200.mjcf.compiler.pack_model (host memory).  precision: B2S_F32 (production) or B2S_F64 (debug). */
int b2s_create(const void* model_blob_host, size_t nbytes, int n_env, int device, int precision, b2s_sim** out);
/* MjSim.free (binding_utils.py:1186-1192) */
void b2s_destroy(b2s_sim* sim);
const char* b2s_last_error(void);
/* all device work of this handle is enqueued on `cuda_stream` (a cudaStream_t); default: the legacy default stream */
int b2s_set_stream(b2s_sim* sim, void* cuda_stream);

/* MjSim.reset -> mj_resetData (binding_utils.py:1089-1091); env_mask: n_env bytes on device (non-zero = reset) or NULL */
int b2s_reset(b2s_sim* sim, const uint8_t* env_mask);
/* MjSim.forward -> mj_forward (binding_utils.py:1093-1095) */
int b2s_forward(b2s_sim* sim);
/* MjSim.step1 / step2 -> mj_step1 / mj_step2 (binding_utils.py:1101-1107); ctrl is read between them */
int b2s_step1(b2s_sim* sim);
int b2s_step2(b2s_sim* sim);
/* MjSim.step -> mj_step (binding_utils.py:1097-1099), repeated n_substeps times inside one kernel with ctrl held */
int b2s_step(b2s_sim* sim, int n_substeps);

/* Named device arrays, leading dimension n_env: qpos qvel qacc qacc_warmstart ctrl time xpos xquat xmat
 * site_xpos site_xmat geom_xpos geom_xmat qM(dense nv x nv) qfrc_bias qfrc_passive qfrc_actuator qfrc_constraint
 * actuator_force ncon contact_geom contact_dist contact_pos contact_frame nefc efc_force warn ...
 * (contact_efc_address, i32 [n_env, maxcon]: each contact's first constraint row, mjContact.efc_address; -1 for a contact without
 * rows - not penetrating, or dropped by the row budget - and for rows ncon .. maxcon - 1)
 * (the attributes the reference touches, SURVEY.md section 8b).  dtype is B2S_F32/F64/I32.  After the first pipeline-mode step also
 * tail_key (i32: each environment's tail cost class) and tail_order (i32: per group, the environment each warp position of the last
 * tail launch ran), the cost order the pipeline's tail hands environments to warps in; written when tail blocks hold 8 warps or more. */
int b2s_array(b2s_sim* sim, const char* name, void** dev_ptr, int* dtype, int* ndim, int64_t shape[4]);

/* MjSim.get_state().flatten() / set_state_from_flattened (binding_utils.py:1155-1184, MjSimState.flatten :56-70): device buffers
 * [n_env, 1 + nq + nv] holding time, qpos, qvel per environment.  b2s_set_state does what the reference does after it: nothing else
 * (call b2s_forward next, as callers of set_state_from_flattened do). */
int b2s_get_state(b2s_sim* sim, void* out_dev);
int b2s_set_state(b2s_sim* sim, const void* in_dev);
/* MjModel.{body,joint,geom,site,actuator,...}_name2id / id2name (binding_utils.py:362-492).  type: "body" "joint" "geom" "site"
 * "actuator" "mesh" "camera" "light".  name2id returns the id or -1 (unknown name / type); id2name returns a pointer that stays valid
 * for the life of the handle, NULL when out of range ("" for unnamed objects). */
int b2s_name2id(const b2s_sim* sim, const char* type, const char* name);
const char* b2s_id2name(const b2s_sim* sim, const char* type, int id);
/* mj_fullM (controllers/parts/controller.py:226-229 builds the dense mass matrix from qM): out_dev [n_env, nv, nv], valid after
 * b2s_forward / b2s_step1, and after b2s_env_step / b2s_step with b2s_set_export or b2s_set_step1_export on */
int b2s_full_m(b2s_sim* sim, void* out_dev);
/* MjData.get_body_jacp/jacr, get_geom_jacp/jacr (binding_utils.py:853-878 and the geom variants): Jacobian of the body frame origin /
 * geom centre (a colliding geom: the others have no pose), [n_env, 3, nv] device buffers (either may be NULL), valid after
 * b2s_forward / b2s_step1, and after b2s_env_step / b2s_step with b2s_set_export or b2s_set_step1_export on */
int b2s_jac_body(b2s_sim* sim, int body_id, void* jacp, void* jacr);
int b2s_jac_geom(b2s_sim* sim, int geom_id, void* jacp, void* jacr);

/* MjData.get_site_jacp/jacr (binding_utils.py:826-852): jacp/jacr are [n_env,3,nv] device buffers (either may be NULL);
 * valid after b2s_forward/b2s_step1, and after b2s_env_step / b2s_step with b2s_set_export or b2s_set_step1_export on. */
int b2s_jac_site(b2s_sim* sim, int site_id, void* jacp, void* jacr);

/* Fused control step = MujocoEnv.step's substep loop (environments/base.py:494-505):
 * n_substeps x { step1 ; controller(action) -> ctrl ; step2 } in ONE kernel with state resident on chip.
 * Configure once with b2s_ctrl_config (fields of controllers/config/default/parts/osc_pose.json + robot indices),
 * then call b2s_env_step(action[n_env, action_dim]) per control step.  obs_out[n_env, obs_dim] may be NULL. */
typedef struct {
  int kind;            /* B2S_CTRL_* */
  int action_dim;      /* arm dims + gripper dims */
  int n_arm;           /* number of arm joints (7) */
  int arm_dof[8];      /* dof (= qvel) index of each arm joint */
  int arm_qpos[8];
  int arm_act[8];      /* actuator index of each arm joint */
  int eef_site;        /* ref_name site id */
  int base_site;       /* "{prefix}{part}_center" site id (controller origin) */
  int n_grip;          /* gripper actuators (2) */
  int grip_act[4];
  double grip_sign[4]; /* format_action signs (models/grippers/panda_gripper.py:55-57) */
  double grip_speed;   /* 0.2 per policy step */
  double kp[6], damping_ratio[6];
  double input_max[6], input_min[6], output_max[6], output_min[6];
  double null_kp;      /* nullspace_torques joint_kp (control_utils.py:7-40), 10 */
  int uncouple_pos_ori;
  int n_obs_site;      /* sites appended to obs (task layer) - reserved */
  /* JOINT_VELOCITY (controllers/parts/generic/joint_vel.py:60-209): per-joint PID gains and action scaling */
  double jv_kp[8], jv_ki[8], jv_kd[8], jv_in_max[8], jv_in_min[8], jv_out_max[8], jv_out_min[8];
  double jv_vel_lo, jv_vel_hi;
  int jv_use_vel_limits, jv_torque_comp;
} b2s_ctrl_cfg;
int b2s_ctrl_config(b2s_sim* sim, const b2s_ctrl_cfg* cfg);
/* impedance_mode of OSC_POSE, OSC_POSITION and JOINT_POSITION, for the controller b2s_ctrl_config configured last (which itself
 * always configures FIXED, so b2s_ctrl_cfg keeps its size and every field its offset).  FIXED uses the gains of b2s_ctrl_cfg.
 * VARIABLE and VARIABLE_KP take the gains from the action at every policy step (osc.py / joint_pos.py set_goal, recalled from
 * robosuite v1.5; no reference checkout was available to check them against).  With d = 6 for both OSC kinds (OSC_POSITION keeps a
 * 6-dim kp and holds orientation with kp[3:6]) and d = n_arm for JOINT_POSITION, and od = 3 / 6 / n_arm delta entries:
 *   VARIABLE     action = [damping_ratio (d), kp (d), delta (od), gripper]   kp = clip(kp, kp_min, kp_max),
 *                                                                           kd = 2 sqrt(kp) clip(damping_ratio, dr_min, dr_max)
 *   VARIABLE_KP  action = [kp (d), delta (od), gripper]                      kp = clip(kp, kp_min, kp_max), kd = 2 sqrt(kp)
 * so action_dim is 2 d + od + 1 or d + od + 1.  The gain parts are only clipped (input_* / output_* scale the delta).  The gains of
 * each environment live in the array "ctrl_gain" [n_env, 16] f64 (kp[8], kd[8]) in both precisions; this call and b2s_ctrl_reset
 * (so b2s_reset_envs) write the configured gains (kd = 2 sqrt(kp) damping_ratio) into it, as the reference rebuilds its controllers
 * at reset.  While a variable mode is configured the array is a snapshot section.  B2S_ERR_ARG: an unknown mode, and in a variable
 * mode: another kind, a limit among the first d entries that is non-finite or negative or has min > max, or an action_dim other than
 * the layout's; the handle then stays in FIXED mode. */
enum { B2S_IMPEDANCE_FIXED = 0, B2S_IMPEDANCE_VARIABLE = 1, B2S_IMPEDANCE_VARIABLE_KP = 2 };
typedef struct {
  int impedance_mode; /* B2S_IMPEDANCE_* */
  double kp_min[8], kp_max[8], damping_ratio_min[8], damping_ratio_max[8];
} b2s_impedance_cfg;
int b2s_ctrl_impedance(b2s_sim* sim, const b2s_impedance_cfg* cfg);
/* controller.reset_goal + update_initial_joints (osc.py:520-544) for masked envs (NULL = all); needs a prior forward */
int b2s_ctrl_reset(b2s_sim* sim, const uint8_t* env_mask);
int b2s_env_step(b2s_sim* sim, const void* action, int n_substeps);
/* MujocoEnv.reset for a device-resident subset (environments/base.py:277-347: _reset_internal -> sim.forward -> controller reset -> observation
 * cache emptied): masked envs (device bytes, NULL = all) take qpos from `qpos_new` ([n_env, nq] device array of the handle's precision holding a
 * sampled initial state for every environment; NULL = qpos0), velocities / accelerations / warm start / ctrl / time / warn cleared, forward pass,
 * controller goals rebuilt, GJK warm starts dropped.  Every launch is asynchronous on the handle's stream: no host round trip, so a horizon-based
 * auto-reset can be enqueued after every step. */
int b2s_reset_envs(b2s_sim* sim, const uint8_t* env_mask, const void* qpos_new);

/* Per-environment world pose of a body welded to the world.  The reference writes sampled placements into the MODEL per reset
 * (Door: `sim.model.body_pos[door_body_id] = door_pos; body_quat = door_quat`, environments/manipulation/door.py:417-427); a batch shares
 * its model constants, so such poses are per-environment DATA here.  After the call the arrays "body_xpos_ov:<id>" [n_env, 3] and
 * "body_xquat_ov:<id>" [n_env, 4] (initialised to the model's pose; fetch them with b2s_array and write them like any state array)
 * replace the constant world pose of that body in every kinematics pass.  Bodies welded to an overridden body keep THEIR constant world
 * pose: override them too (pose = parent pose * local pose).  At most 4 bodies per handle. */
int b2s_body_pose_override(b2s_sim* sim, int body_id);
/* The same override (it takes one of the 4 slots and the same arrays, "body_xpos_ov:<id>" / "body_xquat_ov:<id>"), and in addition every
 * world-welded body below `body_id` that has no override of its own follows it: its pose is (root pose) * (its fixed pose relative to
 * the root), the relative pose composed from the model's local poses in fp64 on the host once, when the call (or any later override)
 * is made.  A body follows its nearest overridden ancestor, and only when that ancestor was registered here.  Moving bodies below
 * such a subtree follow through their parents as always.  Use: a robot's welded root (base, mounts, link0) moved per environment,
 * e.g. to sit behind a table of per-environment length.  Which bodies follow which root is part of the snapshot signature.  A handle
 * without a call here runs exactly the code and arithmetic it ran before. */
int b2s_body_pose_override_tree(b2s_sim* sim, int body_id);

/* Object placement (the reference's UniformRandomSampler / SequentialCompositeSampler.sample, utils/placement_samplers.py, recalled
 * from robosuite v1.5; no reference checkout was available to check it against).  b2s_place_config copies a program of n <= 32
 * entries, one per object in placement order (n = 0 clears it).  It is handle configuration: not a snapshot section, not part of the
 * signature.  b2s_place_objects then places every entry for the masked environments (env_mask: n_env device bytes, NULL = all) in
 * ONE launch on the handle's stream, one warp per environment, without host data.  Entry o of environment e:
 *   base    = base[]                                            when ref = -1
 *           = (x_r, y_r, z_r + ref_dz) of entry ref (< o)      otherwise (ref_dz: the referenced object's top offset when on_top, else 0)
 *   z       = (z_offset + base_z) - bottom_dz                  (bottom_dz: the object's bottom offset when on_top, else 0)
 *   try t   = 0 .. 4999:  x = (x_min + (x_max - x_min) u_x) + base_x,  y likewise with u_y  (the caller has already shrunk the ranges
 *             by the radius for ensure_object_boundary_in_range; an inverted range works as numpy's uniform does)
 *   valid   = not ensure_valid, or for every earlier entry j:
 *             not ( sqrt(dx*dx + dy*dy) <= radius_j + radius  and  z - z_j <= top_j - bottom )
 * The first valid try is taken (lanes evaluate 32 tries per round; the ballot's lowest valid lane is the sequential loop's first
 * success).  Its rotation: pair c = min(floor(u_c * n_rot), n_rot - 1) (0 when n_rot = 1), angle = rot_min[c] + (rot_max[c] -
 * rot_min[c]) u_a, quaternion (cos a/2, sin a/2 * unit axis) w-first about axis 0 / 1 / 2 = x / y / z.  A fixed angle is the pair
 * (a, a); U[0, 2 pi) is (0, 2 pi).
 * Draws: Philox4x32-10 with key = seed, u = 53 bits of two output words formed as in b2s_perturb_model.  Counter (e, counter, o, t):
 * u_x from words (0, 1), u_y from words (2, 3).  Counter (e, counter, o, 0xFFFFFFFF): u_c from words (0, 1), u_a from words (2, 3).
 * Arithmetic in fp64, every operation rounded once (no contraction), in the order written above; sin / cos of a/2 by the library's
 * own fixed sequence (csrc/b2s_place.cuh place_sincos: reduction by pi/2 with fdlibm's split and fdlibm's kernel polynomials), so a
 * host restatement reproduces every bit.  An environment's placement depends only on (seed, counter, e, program).
 * Targets: qpos_adr >= 0 writes qpos[e, qpos_adr .. +7] = (x, y, z, quaternion) of the float64 [n_env, nq] device array `qpos` (the
 * sampled states b2s_reset_envs then takes, converted to the handle's precision by the caller); body >= 0 writes the body's pose
 * override (b2s_body_pose_override) and the override of every overridden body welded to it (at the time of b2s_place_config), as
 * placed pose * pose relative to the body (composed local poses), rounded to the handle's precision last.  Unmasked environments
 * are not written.
 * An environment in which some object has no valid try keeps that object's last try and gets warn bit 1024.  b2s_place_objects leaves
 * the bit pending; the next b2s_reset_envs writes it into `warn` for the environments it resets (it clears every other bit).
 * B2S_ERR_ARG: n outside [0, 32]; in an entry a non-finite field, n_rot outside [1, 8], axis outside [0, 2], ref not -1 or an earlier
 * entry, neither or both of qpos_adr / body, a qpos_adr that is not the first address of a free joint, a body without a pose
 * override, a joint or body placed twice; in b2s_place_objects a counter >= 2^32 or qpos NULL while an entry writes qpos.  Without a
 * program b2s_place_objects does nothing. */
#define B2S_PLACE_MAXROT 8
typedef struct {
  int qpos_adr, body, ref, ensure_valid, axis, n_rot;
  double x_min, x_max, y_min, y_max;
  double base[3], ref_dz, z_offset, bottom_dz;
  double radius, bottom, top; /* horizontal_radius, bottom_offset z, top_offset z */
  double rot_min[B2S_PLACE_MAXROT], rot_max[B2S_PLACE_MAXROT];
} b2s_place;
int b2s_place_config(b2s_sim* sim, const b2s_place* entries_host, int n);
int b2s_place_objects(b2s_sim* sim, double* qpos, const uint8_t* env_mask, uint64_t seed, uint64_t counter);

/* Per-environment model values (domain randomisation; the reference draws e.g. Lift's cube size per model build,
 * environments/manipulation/lift.py:311-314).  Declares a per-environment copy of `field` for object `id`: afterwards the array
 * "<field>:<id>" (fetch it with b2s_array) holds one value per environment, initialised to the model's, and every step reads it.
 *   "geom_size"     [n_env, 3]  colliding sphere / capsule / ellipsoid / cylinder / box geoms
 *   "geom_friction" [n_env, 3]  same geoms
 *   "body_mass"     [n_env]     moving bodies
 *   "body_inertia"  [n_env, 3]  moving bodies: principal moments in the model's inertial frame (body_ipos / body_iquat stay shared)
 *   "dof_damping", "dof_armature", "dof_frictionloss"  [n_env, nv]  id must be -1 (the whole vector); the array is named "<field>".
 *       Damping enters the passive force and the implicit Euler step, armature the mass matrix (and so the derived constants).
 *       Once "dof_frictionloss" is declared, an environment's friction-loss rows are its dofs whose own value is > 0, in dof order;
 *       it needs opt_maxefc >= nv + 8 (B2S_ERR_UNSUPPORTED otherwise).
 * A declared geom (geom_size or geom_friction) also gets "geom_rbound:<id>" [n_env] and "geom_aabb:<id>" [n_env, 6], and its contact
 * parameters "geom_solref:<id>" [n_env, 2] and "geom_solimp:<id>" [n_env, 5], initialised to the model's and read by the contact
 * solref / solimp mixing of every step (they are not fields of their own: they come with the geom's slot).  The first declaration of a handle creates
 * "dof_invweight0" [n_env, nv], "body_invweight0" [n_env, nbody, 2] and "meaninertia" [n_env].  These DERIVED constants start at the
 * model's values and are STALE after a change until b2s_set_const or b2s_reset / b2s_reset_envs (which run the same pass for their
 * masked environments whenever the handle has overrides) recomputes them.  Returns B2S_ERR_ARG for an unknown field or an id out of
 * range, B2S_ERR_UNSUPPORTED for meshes, planes, non-colliding geoms, the world body and bodies welded to it, and beyond 8 geoms or
 * 8 bodies per handle.  Declaring again returns B2S_OK and changes nothing. */
int b2s_model_override(b2s_sim* sim, const char* field, int id);
/* The set-constants pass for the masked environments (env_mask: n_env device bytes, NULL = all), one warp each, on the handle's
 * stream: kinematics and composite inertia at qpos0 (world-pose overrides honoured) -> dof_invweight0, body_invweight0, meaninertia
 * (the compiler's definitions), and the bounding radius / box of every overridden geom from its size.  Environments whose override
 * values are non-finite or non-positive (damping, armature, friction loss: non-finite or negative), whose solref / solimp has a
 * non-finite component, or whose moments violate the triangle inequality, get warn bit 128.  No-op on a handle without overrides. */
int b2s_set_const(b2s_sim* sim, const uint8_t* env_mask);

/* Device perturbation of declared override arrays (dynamics randomisation, the batched counterpart of the reference's DynamicsModder,
 * utils/mjmod.py).  b2s_perturb_config copies a list of (field, id) entries once (n = 0 clears it); every field must already be
 * declared with b2s_model_override.  For the dof fields id -1 perturbs every dof and a dof index that dof alone.
 * b2s_perturb_model then writes every entry of the masked environments (env_mask: n_env device bytes, NULL = all) in ONE launch on the
 * handle's stream, without host data, drawing around the MODEL's value (repeated calls do not random-walk):
 *   B2S_PERTURB_SCALE: v = v_model * (1 + d)     B2S_PERTURB_SHIFT: v = max(0, v_model + d)     d ~ U(-amplitude, amplitude)
 * one_draw = 1 uses one draw for all components of the entry (body_inertia: keeps the triangle inequality).  d comes from
 * Philox4x32-10 with key = seed and counter = (env, counter, entry index, component; 0 with one_draw), u = 53 bits of the first two
 * output words ((w0 >> 5) * 2^26 + (w1 >> 6)) / 2^53, d = amplitude * (2u - 1) in fp64, rounded to the handle's precision last:
 * an environment's values depend only on (seed, counter, env, spec).  The derived constants are NOT updated: they follow at the next
 * b2s_set_const or reset.  B2S_ERR_ARG: undeclared field, negative or non-finite amplitude, amplitude >= 1 in scale mode, counter
 * >= 2^32.  Without a configuration b2s_perturb_model does nothing. */
enum { B2S_PERTURB_SCALE = 0, B2S_PERTURB_SHIFT = 1 };
typedef struct { const char* field; int id; int mode; double amplitude; int one_draw; } b2s_perturb;
int b2s_perturb_config(b2s_sim* sim, const b2s_perturb* spec_host, int n);
int b2s_perturb_model(b2s_sim* sim, const uint8_t* env_mask, uint64_t seed, uint64_t counter);

/* Observation program = MujocoEnv._get_observations flattened (environments/base.py:429-465): one (op, a, b) entry
 * per output scalar (ops: enum OB_* in csrc/b2s_types.cuh; OB_REL_*_LAG entries read the previous sample, as the reference's
 * sensor ordering does: manipulation_env.py:268-329).  Creates the device arrays "obs" [n_env, obs_dim] and "obs_fresh" [n_env]
 * (1 = observation cache empty; set it when an environment is reset).  "obs" is written by b2s_env_step when an observable samples
 * and by b2s_forward for environments whose obs_fresh flag is set.  Without b2s_obs_modifiers every observable samples after the
 * LAST substep of a control step: reset()'s forced update advances the observables' period timer by one model step, so at the
 * control rate every later sample falls on the last substep (utils/observables.py:214-259, environments/base.py:418-427).
 * obs_dim <= 128. */
int b2s_obs_config(b2s_sim* sim, int obs_dim, const int* op_host, const int* a_host, const int* b_host);
/* Sampling rates and corruptors of the observables (Observable.sampling_rate / corruptor, utils/observables.py, with delay 0).
 * row_obs_host[obs_dim] maps each observation row to its observable (0 .. nobs - 1); mods_host[nobs] gives each observable's period
 * T = 1 / sampling_rate in seconds and its corruptor: B2S_CORRUPT_GAUSSIAN (p0 = mean, p1 = std) adds mean + std * z,
 * B2S_CORRUPT_UNIFORM (p0 = min_noise, p1 = max_noise) adds min + (max - min) * u, both then clip to [low, high];
 * B2S_CORRUPT_NONE leaves the value as it is.  Per environment and observable a timer t (fp64), a flag `sampled` and a sample count
 * follow Observable.update after every substep (dt = the model's timestep in fp64):
 *   t += dt;  if not sampled and t <= T: sample, sampled = 1;  if t >= T: sample if not sampled, sampled = 0, t = fmod(t, T)
 * and reset (b2s_forward of an environment whose obs_fresh flag is set) restarts it with t = 0, sampled = 0 and a forced sample.
 * A sample forms the observable's rows as above (poses of this substep's step1, qpos / qvel after its step2) and corrupts them;
 * the rows are the observation cache the lagged entries read.  Noise: Philox4x32-10 with key = seed and counter = (env, the
 * observable's sample count, row, 0), u1 / u2 = 53 bits of output words (0, 1) / (2, 3) as b2s_perturb_model forms u, z by
 * Box-Muller sqrt(-2 log(1 - u1)) cos(2 pi u2), arithmetic in fp64, rounded to the handle's precision last.  Sample counts are never
 * rewound, so episodes do not repeat their noise.  The first call creates "obs_timer" [n_env, nobs] f64, "obs_sampled" [n_env] i32
 * (bit o = observable o) and "obs_nsample" [n_env, nobs] i32; a call on a handle without modifiers (re)starts the timers in the
 * state the default rule has at a control-step boundary (t = dt, sampled).  While configured, the three arrays are snapshot
 * sections.  nobs = 0 clears the configuration (the handle runs exactly as before the first call).  B2S_ERR_ARG: observations not
 * configured, nobs > 32, a non-positive or non-finite period, an unknown corruptor, a non-finite noise parameter, std < 0,
 * max_noise < min_noise, low > high, or a row mapped out of range. */
enum { B2S_CORRUPT_NONE = 0, B2S_CORRUPT_GAUSSIAN = 1, B2S_CORRUPT_UNIFORM = 2 };
typedef struct { double period; int corruptor; double p0, p1, low, high; } b2s_obs_mod;
int b2s_obs_modifiers(b2s_sim* sim, int nobs, const int* row_obs_host, const b2s_obs_mod* mods_host, uint64_t seed);
/* Per-environment object selection (single_object_mode 1 of PickPlace / NutAssembly: pick_place.py, nut_assembly.py draw one object
 * at every reset and switch the observables of the others off).  body_ids_host[n] lists 1 to 4 bodies with a free joint; the call
 * creates "obj_sel" [n_env] i32, zeros at its creation (kept by later calls), which the caller writes (e.g. at a reset).  Observation
 * and task ops OB_SEL_BODY_POS / OB_SEL_BODY_QUAT_XYZW (b = component, quaternion as x, y, z, w) read body body_ids[obj_sel[env]],
 * OB_SEL_INDEX reads obj_sel[env] as a real; every path that writes observations evaluates them (b2s_env_step in all three modes,
 * b2s_forward, b2s_reset_envs).  An environment whose selection is outside [0, n) gets 0 in those rows and warn bit 512; nothing is
 * read through it.  While a list is configured "obj_sel" is a snapshot section and the list is part of the signature.  n = 0 clears
 * the list.  B2S_ERR_ARG: n outside [0, 4], a body without a free joint, or n = 0 while the observation or task table uses a
 * selection op (b2s_obs_config / b2s_task_table in turn refuse such ops while no list is configured). */
int b2s_obs_objects(b2s_sim* sim, int n, const int* body_ids_host);
/* Task outputs "task_out" [n_env,8] = (target body height, |site - body|, grasp flag, horizontal |body - body2|,
 * obj-obj2 contact flag, 0, 0, 0) from the poses/contacts of the
 * last step1 (what the reference's reward()/_check_grasp read: manipulation/lift.py:224-273, manipulation_env.py:331-376).
 * Geom id lists: left / right finger(pad) groups and object geoms. */
int b2s_task_config(b2s_sim* sim, int body, int site, const int* left, int nleft, const int* right, int nright,
                    const int* obj, int nobj);
/* optional second object (Stack's cubeB: staged_rewards, manipulation/stack.py:266-312); call after b2s_task_config */
int b2s_task_config2(b2s_sim* sim, int body2, const int* obj2, int nobj2);
/* optional per-object grasp flags for multi-object tasks (NutAssembly / PickPlace staged_rewards check the grasp against
 * the geoms of the still-active objects: manipulation/nut_assembly.py:318-327, pick_place.py:352-361): up to 4 objects,
 * geoms = concatenated geom id lists, counts[i] = length of list i.  task_out[5] = sum_i 2^i * grasped_i. */
int b2s_task_objects(b2s_sim* sim, int nobjects, const int* geoms, const int* counts);
/* task table: n (<= 64) scalars in the observation-table encoding, evaluated after the LAST substep of b2s_env_step into
 * the array "task_vec" [n_env, n] - the poses reward()/_check_success() read from sim.data after the step
 * (manipulation/door.py:219-266, nut_assembly.py:247-400, pick_place.py:275-425). Requires b2s_obs_config first. */
int b2s_task_table(b2s_sim* sim, int n, const int* op, const int* a, const int* b);

/* Whole-environment snapshots: everything that decides an environment's next control step, as one opaque byte row per environment,
 * so that an environment can be saved mid-episode and resumed, or cloned into others, bit-exactly.  A row is made of named SECTIONS
 * in a fixed order, each 16-byte aligned; the row length is a multiple of 16 bytes.  Sections, each the environment's row of the
 * handle's own array:
 *   always           qpos qvel qacc qacc_warmstart ctrl time, warn (i32), ctrl_goal_pos ctrl_goal_ori ctrl_initial_joint ctrl_grip_state
 *                    ctrl_jv_state ctrl_torque, gjk_cache (npair x 3; written as zeros and ignored on restore while the handle has no
 *                    cache: fused mode before the pipeline's first use, or B2S_NO_GJK_CACHE)
 *   variable impedance  ctrl_gain (f64), while b2s_ctrl_impedance has a variable mode configured; the mode is then part of the signature
 *   b2s_obs_config   obs, obs_fresh (i32), task_out
 *   b2s_obs_modifiers  obs_timer (f64), obs_sampled (i32), obs_nsample (i32), while configured
 *   b2s_task_table   task_vec
 *   b2s_obs_objects  obj_sel (i32), while a list is configured
 *   overrides        body_xpos_ov:<id> body_xquat_ov:<id> per pose override; geom_{size,friction,rbound,aabb,solref,solimp}:<id> per geom
 *                    slot; body_mass:<id> body_inertia:<id> per body slot; the declared dof vectors; dof_invweight0 body_invweight0
 *                    meaninertia (copied, not recomputed: a snapshot taken while they were stale restores them stale)
 * Not in a row: the exported derived arrays (xpos, contacts, efc_*, ...), ncon / nefc / solver_niter, pipeline workspaces,
 * and handle configuration (controller gains, obs / task tables, perturbation tables, observable rates and corruptors).
 * The SIGNATURE is a 64-bit FNV-1a hash of the section table (names, counts, dtypes), the precision, the controller kind, the obs and
 * task op tables and the model blob without its capacity records (opt_maxcon, opt_maxefc and the small-tier pair): rows restore only
 * into a handle with the same signature (the Python layer checks it; the C layer does not).
 * A restored environment continues bit-identically to its source under the same actions given the same library build, precision,
 * mode (b2s_set_mode), B2S_CTRL_SPLIT and B2S_NO_GJK_CACHE, whatever n_env, group count, small tier or neighbours either handle has.
 * b2s_snapshot_info / b2s_snapshot_section describe the layout (name: valid until the next call that changes it). */
int b2s_snapshot_info(b2s_sim* sim, size_t* row_bytes, uint64_t* signature, int* nsections);
int b2s_snapshot_section(b2s_sim* sim, int k, const char** name, int64_t* offset_bytes, int64_t* count, int* dtype);
/* rows_dev [n_rows, row_bytes] <- environment env_index_host[r] for row r (NULL: every environment in order, n_rows == n_env).
 * Indices are checked on the host: one out of range returns B2S_ERR_ARG and enqueues nothing. */
int b2s_snapshot(b2s_sim* sim, void* rows_dev, const int* env_index_host, int n_rows);
/* environment e <- row src_row_dev[e] (device int32 [n_env], e.g. an argmax computed on the device; NULL: row e, n_rows == n_env).
 * -1 leaves the environment untouched; an index >= n_rows or < -1 leaves it untouched and sets warn bit 256.  No physics runs: the
 * exported derived arrays stay stale until the next forward / step (a forward pass would also rewrite qacc, which is observed).  In
 * pipeline / unit-queue mode the call first creates the GJK cache if the handle has none yet, so that it is restored.  Clone = snapshot
 * every environment, then restore with a source map.  Both calls are enqueued on the handle's stream without a host synchronisation. */
int b2s_restore(b2s_sim* sim, const void* rows_dev, int n_rows, const int* src_row_dev);

/* b2s_env_step also exports the derived arrays of its last substep (xpos, contacts, efc ...) when flag != 0 (default 1);
 * the throughput path switches it off so that per-step HBM traffic is state + action + obs only */
int b2s_set_export(b2s_sim* sim, int flag);

/* Contact geometry without the full export (what check_contact / get_contacts / _check_grasp read from data.contact after
 * env.step, utils/sim_utils.py, manipulation_env.py).  flag != 0 (default 0): the LAST substep of every b2s_env_step / b2s_step call
 * writes ncon [n_env] and contact_geom [n_env, maxcon, 2], contact_dim, contact_dist, contact_pos [.., 3], contact_frame [.., 9] and
 * contact_friction [.., 3]: the contacts of that substep's step1 in static-pair order (data.contact[:ncon] after mj_step with
 * lite_physics), rows ncon .. maxcon - 1 with geom -1 and zeros.  All three schedules write the same bits, so b2s_env_step keeps the
 * handle's mode (b2s_set_export = 1, which also writes these arrays, still runs the fused kernel).  The arrays are valid once the
 * call's work on the handle's stream is done.  b2s_reset_envs writes the forward pass's contacts of the masked environments (with or
 * without the flag, as b2s_forward does for all); after b2s_restore they are stale until the next step, like the other derived
 * arrays.  They are not a snapshot section, and neither they nor the flag are part of the signature.  B2S_ERR_ARG: null handle. */
int b2s_set_contact_export(b2s_sim* sim, int flag);

/* The step-1 arrays without the full export (what reward / success code, controllers and safety filters read from sim.data after
 * env.step: body_xpos, get_site_xpos / xmat, get_site_jacp / jacr, mj_fullM).  flag != 0 (default 0): the LAST substep of every
 * b2s_env_step / b2s_step call writes xpos [n_env, nbody, 3], xquat [.., 4], xmat [.., 9], site_xpos [n_env, nsite, 3], site_xmat
 * [.., 9], geom_xpos [n_env, ngeom, 3] / geom_xmat [.., 9] of the colliding geoms, qM [n_env, nv, nv], cdof [n_env, nv, 6],
 * qfrc_bias [n_env, nv] and qfrc_passive [n_env, nv]: the values of that substep's step1 (mj_step's position and velocity stages),
 * the same bits in all three schedules, so b2s_env_step keeps the handle's mode (b2s_set_export = 1, which also writes these arrays,
 * still runs the fused kernel).  The poses of non-colliding (visual) geoms are never computed: their rows keep whatever they held.
 * The arrays are valid once the call's work on the handle's stream is done, and b2s_jac_site / b2s_jac_body / b2s_jac_geom and
 * b2s_full_m, which read them, are then valid too.  b2s_reset_envs writes them for the masked environments (with or without the
 * flag, through its forward pass, as b2s_forward does for all); after b2s_restore they are stale until the next step, like the
 * other derived arrays.  They are not a snapshot section, and neither they nor the flag are part of the signature.  B2S_ERR_ARG:
 * null handle. */
int b2s_set_step1_export(b2s_sim* sim, int flag);

/* The step-2 arrays without the full export (what energy penalties, smoothness terms and contact-force rewards or safety checks
 * read from sim.data after env.step: actuator_force, qfrc_actuator, qacc, efc_force through mj_contactForce).  flag != 0 (default
 * 0): the LAST substep of every b2s_env_step / b2s_step call writes qfrc_actuator, qfrc_smooth, qacc_smooth, qfrc_constraint
 * [n_env, nv], actuator_force [n_env, nu], nefc [n_env], efc_type (i32), efc_D, efc_R, efc_aref, efc_force [n_env, maxefc] (zeros
 * from row nefc on), efc_J [n_env, maxefc, nv] (the first nefc * nv values of the row; the rest keep whatever they held),
 * solver_niter [n_env] and contact_efc_address [n_env, maxcon]: the values of that substep's constraint stage and step2 (mj_step's
 * forward dynamics and constraint solve), the same bits in all three schedules, so b2s_env_step keeps the handle's mode
 * (b2s_set_export = 1, which also writes these arrays, still runs the fused kernel).  The arrays are valid once the call's work on
 * the handle's stream is done.  b2s_reset_envs writes them for the masked environments (with or without the flag, through its
 * forward pass, as b2s_forward does for all); after b2s_restore they are stale until the next step, like the other derived arrays.
 * qacc is state and is written by every step.  They are not a snapshot section, and neither they nor the flag are part of the
 * signature.  B2S_ERR_ARG: null handle. */
int b2s_set_step2_export(b2s_sim* sim, int flag);

/* Scheduling of b2s_env_step / b2s_step: 0 = fused (one kernel per call, state resident in shared memory for all
 * substeps), 1 = pipeline (per substep and environment group: phase 0, phase 1 (narrow phase + controller), the tail kernel and,
 * when the model has a small tail tier, its large-tier re-run, exchanging a workspace row through L2; one CUDA graph per group,
 * replayed on the group's own stream), 2 = unit queue (one persistent kernel per control step).  Results are identical; see
 * DESIGN.md sections 4 and 5 for when each wins. */
int b2s_set_mode(b2s_sim* sim, int mode);

/* number of kernels this handle has launched since creation (bench.py "gpu_launches") */
int64_t b2s_launch_count(const b2s_sim* sim);

/* Host-only diagnostic (no device needed): words per warp of the shared-memory layouts and of the global workspace row that a model
 * of these dimensions gets - out_words[5] = fused kernel, phase 0, tail small tier, tail large tier, row.  out_layouts / out_pio may
 * be NULL; see csrc/b2s_capi.cu for their packing (tests/test_cpu_layouts.py checks the layout invariants with them). */
int b2s_debug_layouts(int nq, int nv, int nu, int nbody, int ncg, int nsite, int hc_stride, int maxcon, int maxefc, int mc_small,
                      int me_small, int osc_in_tail, int* out_words, int* out_layouts, int* out_pio);

#ifdef __cplusplus
}
#endif
#endif
