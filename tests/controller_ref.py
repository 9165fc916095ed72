"""Independent fp64 restatement of the reference's arm and gripper controllers, in numpy, from the reference's semantics (the
file:line citations are robosuite v1.5.2's).  It is the yardstick of tests/test_cpu_controllers.py (against the reference's own
records and the CPU oracle) and tests/test_gpu_controllers.py (against the device, substep by substep).

  Controller.scale_action                                  controllers/parts/controller.py:149-168
  OperationalSpaceController.set_goal / run_controller     controllers/parts/arm/osc.py:225-283, 403-495 (kind 1 OSC_POSE, 5 OSC_POSITION)
  opspace_matrices / nullspace_torques / orientation_error utils/control_utils.py:7-111 (np.linalg.pinv, rcond 1e-15)
  axisangle2quat / quat2mat (float32)                      utils/transform_utils.py:461-487, 515-538
  JointVelocityController                                  controllers/parts/generic/joint_vel.py:129-209 (kind 2; RingBuffer
                                                           utils/buffers.py), the constructor's `torque_compensation` read as
                                                           `use_torque_compensation` (joint_tor.py:109)
  JointPositionController (delta, fixed impedance)         controllers/parts/generic/joint_pos.py:160-262 (kind 3)
  JointTorqueController                                    controllers/parts/generic/joint_tor.py:112-160 (kind 4)
  PandaGripper / RethinkGripper.format_action              models/grippers/panda_gripper.py:43-58, rethink_gripper.py:43-58
  SimpleGripController.run_controller                      controllers/parts/gripper/simple_grip.py:150-186
  FixedBaseRobot.control (clip to ctrlrange)               robots/fixed_base_robot.py:149-153

One call is one controller evaluation between step 1 and step 2 of a substep; `action` is given on the policy substep only.

Inputs (fp64 or anything numpy casts to it): `inp` holds one environment's qpos [nq], qvel [nv], site_xpos [nsite, 3], site_xmat
[nsite, 9], cdof [nv, 6] (spatial motion axes [angular; linear at the world origin], the engine's convention), qM [nv, nv] (dense)
and qfrc_bias [nv].  Site Jacobians are formed from cdof, site velocities are J_site @ qvel.  `state` holds the controller state in
the device's per-environment layout: goal_pos [3] and goal_ori [9] (base frame), initial_joint [8], grip [4] (the grippers'
integrated actions) and jv [72] (joint controllers: goal [0:8], last error [8:16], summed error [16:24], the derivative ring
[24:64] as 5 rows of 8, ring pointer [64], ring size [65], saturation flag [66]).

Returns dict(torque [n_arm] before the clip, ctrl [nu] (the arm and gripper actuators; other entries 0), state (the new state))."""
import numpy as np

STATE_SIZES = {"goal_pos": 3, "goal_ori": 9, "initial_joint": 8, "grip": 4, "jv": 72}
EPS4 = np.finfo(float).eps * 4.0  # transform_utils.EPS


def scale_action(a, in_max, in_min, out_max, out_min):
    """Controller.scale_action: clip to the input range, then the affine map onto the output range"""
    a = np.clip(np.asarray(a, dtype=np.float64), in_min, in_max)
    scale = np.abs(out_max - out_min) / np.abs(in_max - in_min)
    return (a - (in_max + in_min) / 2.0) * scale + (out_max + out_min) / 2.0


def delta_rotation(aa):
    """quat2mat(axisangle2quat(aa)): the quaternion is rounded to float32 and the matrix formed in float32, as the reference does"""
    aa = np.asarray(aa, dtype=np.float64)
    angle = np.linalg.norm(aa)
    if angle == 0.0:  # math.isclose(angle, 0.0) with its default tolerances
        qxyzw = np.array([0.0, 0.0, 0.0, 1.0])
    else:
        qxyzw = np.concatenate([aa / angle * np.sin(angle / 2.0), [np.cos(angle / 2.0)]])
    q = qxyzw.astype(np.float32)[[3, 0, 1, 2]]
    n = np.float32(np.dot(q, q))
    if n < EPS4:
        return np.identity(3)
    q = q * np.float32(np.sqrt(np.float64(np.float32(2.0) / n)))
    q2 = np.outer(q, q)
    one = np.float32(1.0)
    return np.array([[one - q2[2, 2] - q2[3, 3], q2[1, 2] - q2[3, 0], q2[1, 3] + q2[2, 0]],
                     [q2[1, 2] + q2[3, 0], one - q2[1, 1] - q2[3, 3], q2[2, 3] - q2[1, 0]],
                     [q2[1, 3] - q2[2, 0], q2[2, 3] + q2[1, 0], one - q2[1, 1] - q2[2, 2]]], dtype=np.float32).astype(np.float64)


def orientation_error(desired, current):
    """control_utils.orientation_error: half the sum of the column cross products"""
    return 0.5 * sum(np.cross(current[:, k], desired[:, k]) for k in range(3))


def chain_dofs(model, body):
    """the dofs that move `body`: those of the body and of its ancestors"""
    out = []
    while body > 0:
        out += [d for d in range(model.nv) if int(model.dof_bodyid[d]) == body]
        body = int(model.body_parentid[body])
    return sorted(out)


def site_jacobian(model, cdof, site, point):
    """[jacp; jacr] [6, nv] of a point fixed to the site's body (mj_jacSite)"""
    J = np.zeros((6, model.nv))
    for d in chain_dofs(model, int(model.site_bodyid[site])):
        ang, lin = cdof[d, :3], cdof[d, 3:]
        J[:3, d] = lin + np.cross(ang, point)
        J[3:, d] = ang
    return J


def _lo_hi(model, u):
    return float(model.actuator_ctrlrange[u, 0]), float(model.actuator_ctrlrange[u, 1])


def _grippers(model, cfg, st, ctrl, ga):
    """format_action (policy substeps: integrate sign(a) * speed, clipped to [-1, 1]) and SimpleGripController: the midpoint of
    ctrlrange plus half its width times the integrated action, clipped to ctrlrange"""
    for g in range(cfg.n_grip):
        if ga is not None:
            st["grip"][g] = np.clip(st["grip"][g] + cfg.grip_sign[g] * cfg.grip_speed * np.sign(ga), -1.0, 1.0)
        u = cfg.grip_act[g]
        lo, hi = _lo_hi(model, u)
        ctrl[u] = np.clip(0.5 * (hi + lo) + 0.5 * (hi - lo) * st["grip"][g], lo, hi)


def _arm_out(model, cfg, torque, ctrl):
    for k in range(cfg.n_arm):
        u = cfg.arm_act[k]
        ctrl[u] = np.clip(torque[k], *_lo_hi(model, u))


def _osc(model, cfg, inp, st, action, ctrl):
    na = cfg.n_arm
    dofs = [cfg.arm_dof[k] for k in range(na)]
    qadr = [cfg.arm_qpos[k] for k in range(na)]
    spos, smat = inp["site_xpos"], inp["site_xmat"].reshape(-1, 3, 3)
    ref_pos, ref_ori = spos[cfg.eef_site], smat[cfg.eef_site]
    org_pos, org_ori = spos[cfg.base_site], smat[cfg.base_site]
    if action is not None:
        od = 3 if cfg.kind == 5 else 6  # OSC_POSITION: a 3-dim arm action, the orientation goal re-anchored (zero delta)
        lim = [np.array([getattr(cfg, f)[k] for k in range(od)]) for f in ("input_max", "input_min", "output_max", "output_min")]
        sd = np.zeros(6)
        sd[:od] = scale_action(action[:od], *lim)
        # goal in the base frame: the current eef pose in that frame moved by the delta (input_ref_frame "base")
        st["goal_pos"][:] = org_ori.T @ (ref_pos - org_pos) + sd[:3]
        st["goal_ori"][:] = (delta_rotation(sd[3:]) @ (org_ori.T @ ref_ori)).reshape(9)
        ga = action[od]
    else:
        ga = None
    Jf = site_jacobian(model, inp["cdof"], cfg.eef_site, ref_pos)
    Jb = site_jacobian(model, inp["cdof"], cfg.base_site, org_pos)
    vel = (Jf - Jb) @ inp["qvel"]  # eef velocity relative to the controller's origin site (zero for a fixed base)
    des_pos = org_ori @ st["goal_pos"] + org_pos
    des_ori = org_ori @ st["goal_ori"].reshape(3, 3)
    err = np.concatenate([des_pos - ref_pos, orientation_error(des_ori, ref_ori)])
    kp = np.array([cfg.kp[k] for k in range(6)])
    kd = 2.0 * np.sqrt(kp) * np.array([cfg.damping_ratio[k] for k in range(6)])
    F = kp * err - kd * vel
    # opspace_matrices
    J = Jf[:, dofs]
    M = inp["qM"][np.ix_(dofs, dofs)]
    Mi = np.linalg.inv(M)
    lam_full = np.linalg.pinv(J @ Mi @ J.T, rcond=1e-15)
    if cfg.uncouple_pos_ori:
        lam_pos = np.linalg.pinv(J[:3] @ Mi @ J[:3].T, rcond=1e-15)
        lam_ori = np.linalg.pinv(J[3:] @ Mi @ J[3:].T, rcond=1e-15)
        wrench = np.concatenate([lam_pos @ F[:3], lam_ori @ F[3:]])
    else:
        wrench = lam_full @ F
    Jbar = Mi @ J.T @ lam_full
    N = np.eye(na) - Jbar @ J
    # nullspace_torques: posture toward the initial joints with kp = null_kp, kv = 2 sqrt(kp)
    q, qd = inp["qpos"][qadr], inp["qvel"][dofs]
    pose = M @ (cfg.null_kp * (st["initial_joint"][:na] - q) - 2.0 * np.sqrt(cfg.null_kp) * qd)
    torque = J.T @ wrench + inp["qfrc_bias"][dofs] + N.T @ pose
    _arm_out(model, cfg, torque, ctrl)
    _grippers(model, cfg, st, ctrl, ga)
    return torque


def _joint_scale(cfg, a):
    na = cfg.n_arm
    lim = [np.array([getattr(cfg, f)[k] for k in range(na)]) for f in ("jv_in_max", "jv_in_min", "jv_out_max", "jv_out_min")]
    return scale_action(a[:na], *lim)


def _jv(model, cfg, inp, st, action, ctrl):
    na = cfg.n_arm
    dofs = [cfg.arm_dof[k] for k in range(na)]
    jv = st["jv"]
    if action is not None:  # set_goal
        goal = _joint_scale(cfg, action)
        if cfg.jv_use_vel_limits:
            goal = np.clip(goal, cfg.jv_vel_lo, cfg.jv_vel_hi)
        jv[:na] = goal
    goal = jv[:na]
    ring = jv[24:64].reshape(5, 8)
    err = goal - inp["qvel"][dofs]
    derr = err - jv[8:8 + na]
    jv[8:8 + na] = err
    ptr = (int(jv[64]) + 1) % 5  # RingBuffer.push
    ring[ptr, :na] = derr
    size = min(int(jv[65]) + 1, 5)
    jv[64], jv[65] = ptr, size
    if not jv[66]:
        jv[16:16 + na] += err
    kp, ki, kd = (np.array([getattr(cfg, f)[k] for k in range(na)]) for f in ("jv_kp", "jv_ki", "jv_kd"))
    torque = kp * err + ki * jv[16:16 + na] + kd * ring[:size, :na].mean(axis=0)
    if cfg.jv_torque_comp:
        torque = torque + inp["qfrc_bias"][dofs]
    _arm_out(model, cfg, torque, ctrl)
    clipped = np.array([ctrl[cfg.arm_act[k]] for k in range(na)])
    jv[66] = 0.0 if np.sum(np.abs(clipped - torque)) == 0 else 1.0
    _grippers(model, cfg, st, ctrl, None if action is None else action[na])
    return torque


def _jp(model, cfg, inp, st, action, ctrl):
    na = cfg.n_arm
    dofs = [cfg.arm_dof[k] for k in range(na)]
    q = inp["qpos"][[cfg.arm_qpos[k] for k in range(na)]]
    jv = st["jv"]
    if action is not None:  # delta input: the goal is the current joint positions moved by the scaled action
        jv[:na] = q + _joint_scale(cfg, action)
    kp, kd = (np.array([getattr(cfg, f)[k] for k in range(na)]) for f in ("jv_kp", "jv_kd"))
    desired = kp * (jv[:na] - q) - kd * inp["qvel"][dofs]
    if cfg.jv_torque_comp:
        torque = inp["qM"][np.ix_(dofs, dofs)] @ desired + inp["qfrc_bias"][dofs]
    else:
        torque = desired
    _arm_out(model, cfg, torque, ctrl)
    _grippers(model, cfg, st, ctrl, None if action is None else action[na])
    return torque


def _jt(model, cfg, inp, st, action, ctrl):
    na = cfg.n_arm
    dofs = [cfg.arm_dof[k] for k in range(na)]
    jv = st["jv"]
    if action is not None:  # the goal torque is clipped to the torque limits (the actuators' ctrlrange)
        lo, hi = np.array([_lo_hi(model, cfg.arm_act[k]) for k in range(na)]).T
        jv[:na] = np.clip(_joint_scale(cfg, action), lo, hi)
    torque = jv[:na] + (inp["qfrc_bias"][dofs] if cfg.jv_torque_comp else 0.0)
    _arm_out(model, cfg, torque, ctrl)
    _grippers(model, cfg, st, ctrl, None if action is None else action[na])
    return torque


def run(model, cfg, inp, state, action=None):
    """one controller evaluation (see the module docstring); `state` is not modified"""
    inp = {k: np.asarray(v, dtype=np.float64) for k, v in inp.items()}
    st = {k: np.array(state[k], dtype=np.float64).reshape(n) for k, n in STATE_SIZES.items()}
    action = None if action is None else np.asarray(action, dtype=np.float64)
    ctrl = np.zeros(model.nu)
    fn = {1: _osc, 5: _osc, 2: _jv, 3: _jp, 4: _jt}[int(cfg.kind)]
    torque = fn(model, cfg, inp, st, action, ctrl)
    return dict(torque=np.asarray(torque, dtype=np.float64), ctrl=ctrl, state=st)


def run_given_goal(model, cfg, inp, state, action, goal_ori):
    """run(), except that for the OSC kinds on a policy substep the torques and ctrl are those of the orientation goal `goal_ori`,
    the one another implementation's set_goal produced.  The delta rotation is formed in float32 (transform_utils.quat2mat), and
    numpy's BLAS, the C oracle and the device's contracted float32 arithmetic each round it their own way in the last float32 bit;
    that alone moves the torques by ~kp * 1e-7.  So the goal is compared at float32 precision on its own (it is returned as run()
    formed it, in `state`), and the torques are judged on the same goal at fp64 precision."""
    r = run(model, cfg, inp, state, action)
    if action is None or cfg.kind not in (1, 5):
        return r
    st = {k: v.copy() for k, v in r["state"].items()}
    st["goal_ori"] = np.asarray(goal_ori, dtype=np.float64).reshape(9)
    r2 = run(model, cfg, inp, st, None)
    return dict(torque=r2["torque"], ctrl=r2["ctrl"], state=r["state"])


KIND_NAMES = {1: "OSC_POSE", 2: "JOINT_VELOCITY", 3: "JOINT_POSITION", 4: "JOINT_TORQUE", 5: "OSC_POSITION"}


def make_config(model, robot, kind, cls, **part):
    """controller_config.resolve of the reference's default part config of `kind` (1-5) for `robot` ("Panda" / "Sawyer"), with
    the part config's keys overridden by `part` (e.g. uncouple_pos_ori, use_torque_compensation, velocity_limits), into `cls`
    (the engine's or the oracle's CtrlCfg)"""
    from robosuite_b200 import controller_config as cc

    arm = cc.load_part_controller_config(KIND_NAMES[kind])
    arm.update(part)
    comp = cc.refactor_composite_controller_config(arm, robot, ["right"])
    return cc.resolve(model, comp, cls, gripper="rethink" if robot == "Sawyer" else "panda")


# ---- test cases shared by the CPU and GPU tests: one arm pose, controller state and action per case
ARM_HOME = {"Panda": np.array([0, np.pi / 16.0, 0.00, -np.pi / 2.0 - np.pi / 3.0, 0.00, np.pi - 0.2, np.pi / 4]),
            "Sawyer": np.array([0, -1.18, 0.0, 2.18, 0.0, 0.57, -1.57])}
# Panda with joints 2, 4 and 6 at 0: joints 1, 3, 5 and 7 share one axis, J loses rank and the smallest eigenvalue of
# J M^-1 J^T is ~1e-17 of the largest, below pinv's cut-off.  Joint 4 moved off 0 by 1e-3 / 1e-5 / 1e-7 puts it at about
# 2e-7 / 2e-11 / 2e-15: well inside, at the fast-path switch of b2s_oscmath.h (1e-11), and just above the cut-off.  Every joint
# value is exactly representable in fp32.
SINGULAR = np.array([0.25, 0.0, 0.125, 0.0, 0.0625, 0.0, 0.5])
NEAR = {"near_1e-3": 1e-3, "near_1e-5": 1e-5, "near_1e-7": 1e-7}
CASES = ("ordinary", "beyond_range", "grip_saturated", "clip", "singular") + tuple(NEAR)
PANDA_ONLY = ("singular",) + tuple(NEAR)


def case_arm(robot, case, rng):
    """(arm joint positions, arm joint velocities) of a case"""
    if case in PANDA_ONLY:
        q = SINGULAR.copy()
        q[3] = NEAR.get(case, 0.0)
        return q, np.array([0.1, -0.2, 0.15, 0.05, -0.1, 0.2, -0.3]) * rng.uniform(0.5, 1.5)
    q = ARM_HOME[robot] + rng.normal(0, 0.05, 7)
    return q, rng.normal(0, 3.0 if case == "clip" else 0.2, 7)


def case_state(model, cfg, case, rng, site_xpos, site_xmat, qpos):
    """a controller state for a case, from the current site poses and qpos: goals near the current eef pose in the base frame
    (far from it for "clip"), a gripper integrator near its limits for "grip_saturated", and a joint-controller state with a
    filled, mid-cycle derivative ring"""
    ref_pos, ref_ori = site_xpos[cfg.eef_site], site_xmat[cfg.eef_site].reshape(3, 3)
    org_pos, org_ori = site_xpos[cfg.base_site], site_xmat[cfg.base_site].reshape(3, 3)
    far = case == "clip"
    st = {"goal_pos": org_ori.T @ (ref_pos - org_pos) + rng.normal(0, 0.3 if far else 0.02, 3),
          "goal_ori": (delta_rotation(rng.normal(0, 1.0 if far else 0.1, 3)) @ org_ori.T @ ref_ori).reshape(9),
          "initial_joint": np.zeros(8), "grip": np.zeros(4), "jv": np.zeros(72)}
    na = cfg.n_arm
    qa = qpos[[cfg.arm_qpos[k] for k in range(na)]]
    st["initial_joint"][:na] = qa + rng.normal(0, 0.1, na)
    st["grip"][:cfg.n_grip] = rng.choice([-0.95, 0.95], cfg.n_grip) if case == "grip_saturated" else rng.uniform(-1, 1, cfg.n_grip)
    jv = st["jv"]
    if cfg.kind == 2:
        jv[:na] = rng.uniform(-1, 1, na)
        jv[8:8 + na] = rng.normal(0, 0.3, na)
        jv[16:16 + na] = rng.normal(0, 3.0, na)
        jv[24:64].reshape(5, 8)[:, :na] = rng.normal(0, 0.1, (5, na))
        jv[64], jv[65], jv[66] = rng.integers(0, 5), rng.integers(0, 6), rng.integers(0, 2)
    elif cfg.kind == 3:
        jv[:na] = qa + rng.normal(0, 0.5 if far else 0.03, na)
    elif cfg.kind == 4:
        jv[:na] = rng.uniform(-3, 3, na)
    return st


def case_action(cfg, case, rng):
    a = rng.uniform(-1, 1, cfg.action_dim)
    if case == "beyond_range":
        a[:-1] = rng.choice([-1.7, 1.7], cfg.action_dim - 1) * rng.uniform(1, 2, cfg.action_dim - 1)
        a[-1] = 0.0
    elif case == "grip_saturated":
        a[-1] = 2.0 if rng.integers(0, 2) else -2.0
    elif case == "clip":
        a[:-1] = np.sign(a[:-1]) * 1.5
    return a


def controlled_actuators(cfg):
    """the actuators whose ctrl the controller writes"""
    return [cfg.arm_act[k] for k in range(cfg.n_arm)] + [cfg.grip_act[g] for g in range(cfg.n_grip)]
