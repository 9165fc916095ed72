"""controller_config plugin surface -> fused-controller configuration.

Accepts the reference's composite controller JSON/dict schema unchanged
(`robosuite/controllers/config/robots/default_panda.json`, `config/default/parts/osc_pose.json`; selection logic
`robosuite/controllers/parts/controller_factory.py:145-159`) and resolves the model indices the way
`robosuite/robots/robot.py:302-332,911-979` does (joint / actuator / site name lookups by naming prefix).

OSC_POSE, OSC_POSITION and JOINT_POSITION take `impedance_mode` "fixed", "variable" or "variable_kp" with `kp_limits` and
`damping_ratio_limits`: in the variable modes the policy sets the gains at every control step through the action (see `_impedance`
for the layout; `action_dim` and `BatchedMujocoEnv.action_spec` follow it).  Not implemented, with NotImplementedError: absolute
inputs, `input_ref_frame` "world", interpolators and `qpos_limits`.
"""
import json
import os

import numpy as np

_DEFAULT_OSC_POSE = {
    "type": "OSC_POSE", "input_max": 1, "input_min": -1,
    "output_max": [0.05, 0.05, 0.05, 0.5, 0.5, 0.5], "output_min": [-0.05, -0.05, -0.05, -0.5, -0.5, -0.5],
    "kp": 150, "damping_ratio": 1, "impedance_mode": "fixed", "kp_limits": [0, 300], "damping_ratio_limits": [0, 10],
    "position_limits": None, "orientation_limits": None, "uncouple_pos_ori": True, "input_type": "delta",
    "input_ref_frame": "base", "interpolation": None, "ramp_ratio": 0.2,
}

# gripper format_action sign patterns and speed (models/grippers/panda_gripper.py:43-58, rethink_gripper.py:56)
GRIPPER_SIGNS = {"panda": [-1.0, 1.0], "rethink": [1.0, -1.0]}
GRIPPER_SPEED = {"panda": 0.2, "rethink": 0.2}


def default_composite_config(robot="Panda"):
    """Same content as config/robots/default_{panda,sawyer}.json: BASIC composite, OSC_POSE arm, GRIP gripper."""
    part = dict(_DEFAULT_OSC_POSE)
    part["gripper"] = {"type": "GRIP"}
    return {"type": "BASIC", "body_parts": {"arms": {"right": part}}}


def load_composite_controller_config(controller=None, robot="Panda"):
    """Mirror of composite_controller_factory.load_composite_controller_config (:73-138): None -> robot default,
    a path -> JSON file, a dict -> used as is."""
    if controller is None:
        return default_composite_config(robot)
    if isinstance(controller, dict):
        return controller
    if isinstance(controller, str) and os.path.exists(controller):
        with open(controller) as f:
            return json.load(f)
    raise ValueError(f"unknown controller config {controller!r}")


def _arr6(v):
    a = np.asarray(v, dtype=np.float64)
    return np.full(6, float(a)) if a.ndim == 0 else a.astype(np.float64)


_DEFAULT_JOINT_VELOCITY = {"type": "JOINT_VELOCITY", "input_max": 1, "input_min": -1, "output_max": 0.5, "output_min": -0.5,
                           "kp": 3.0, "velocity_limits": [-1, 1], "interpolation": None, "ramp_ratio": 0.2}


# controllers/config/default/parts/osc_position.json
_DEFAULT_OSC_POSITION = {"type": "OSC_POSITION", "input_max": 1, "input_min": -1, "output_max": [0.05, 0.05, 0.05],
                         "output_min": [-0.05, -0.05, -0.05], "kp": 150, "damping_ratio": 1, "impedance_mode": "fixed",
                         "kp_limits": [0, 300], "damping_ratio_limits": [0, 10], "position_limits": None, "input_type": "delta",
                         "input_ref_frame": "base", "interpolation": None, "ramp_ratio": 0.2}
# controllers/config/default/parts/joint_position.json, joint_torque.json
_DEFAULT_JOINT_POSITION = {"type": "JOINT_POSITION", "input_max": 1, "input_min": -1, "output_max": 0.05, "output_min": -0.05,
                           "kp": 50, "damping_ratio": 1, "impedance_mode": "fixed", "kp_limits": [0, 300],
                           "damping_ratio_limits": [0, 10], "qpos_limits": None, "interpolation": None, "ramp_ratio": 0.2}
_DEFAULT_JOINT_TORQUE = {"type": "JOINT_TORQUE", "input_max": 1, "input_min": -1, "output_max": 0.1, "output_min": -0.1,
                         "torque_limits": None, "interpolation": None, "ramp_ratio": 0.2}


def load_part_controller_config(default_controller="OSC_POSE"):
    """suite.load_part_controller_config(default_controller=...) (controllers/parts/controller_factory.py:16-70)"""
    table = {"OSC_POSE": _DEFAULT_OSC_POSE, "OSC_POSITION": _DEFAULT_OSC_POSITION, "JOINT_VELOCITY": _DEFAULT_JOINT_VELOCITY,
             "JOINT_POSITION": _DEFAULT_JOINT_POSITION, "JOINT_TORQUE": _DEFAULT_JOINT_TORQUE}
    if default_controller not in table:
        raise NotImplementedError(f"part controller {default_controller} is not implemented")
    return dict(table[default_controller])


def refactor_composite_controller_config(part_cfg, robot_type="Panda", arms=("right",)):
    """old-style part config -> BASIC composite config (composite_controller_factory.py:40-70)"""
    part = dict(part_cfg)
    part.setdefault("gripper", {"type": "GRIP"})
    return {"type": "BASIC", "body_parts": {"arms": {arms[0]: part}}}


def _arr(v, n):
    a = np.asarray(v, dtype=np.float64)
    return np.full(n, float(a)) if a.ndim == 0 else a.astype(np.float64)


# impedance_mode (osc.py, joint_pos.py IMPEDANCE_MODES) -> b2s_ctrl_cfg.impedance_mode (B2S_IMPEDANCE_*); the arm kinds that have one
IMPEDANCE_MODES = {"fixed": 0, "variable": 1, "variable_kp": 2}
IMPEDANCE_KINDS = ("OSC_POSE", "OSC_POSITION", "JOINT_POSITION")


def _impedance(c, arm, d, od):
    """impedance_mode, the gain limits (nums2array: broadcast to d = 6 for OSC, n_arm for JOINT_POSITION) and action_dim: the
    action is [damping_ratio (d), kp (d), delta (od), gripper] in "variable" mode, [kp (d), delta (od), gripper] in "variable_kp",
    [delta (od), gripper] in "fixed".  These layouts and the clip of the gains are recalled from robosuite v1.5 (osc.py,
    joint_pos.py set_goal / control_limits); no reference checkout was available to check them against."""
    mode = IMPEDANCE_MODES[arm.get("impedance_mode", "fixed")]
    c.action_dim = (0 if mode == 0 else d if mode == 2 else 2 * d) + od + 1
    if mode == 0:
        return
    if "impedance_mode" not in (f for f, _ in type(c)._fields_):
        raise NotImplementedError(f"{type(c).__name__} has no variable impedance fields")
    kpl, drl = arm.get("kp_limits", [0, 300]), arm.get("damping_ratio_limits", [0, 10])
    lim = [_arr(kpl[0], d), _arr(kpl[1], d), _arr(drl[0], d), _arr(drl[1], d)]
    c.impedance_mode = mode
    for name, v in zip(("kp_min", "kp_max", "damping_ratio_min", "damping_ratio_max"), lim):
        if v.shape != (d,):
            raise ValueError(f"{name}: expected a scalar or {d} values, got {v.shape}")
        for k in range(d):
            getattr(c, name)[k] = v[k]


def resolve(model, composite_cfg, cfg_struct_cls, robot_prefix="robot0_", gripper_prefix="gripper0_right_", gripper="panda"):
    """Build the C struct (engine.CtrlCfg or the oracle's CtrlCfg: same layout) for one fixed-base arm + gripper."""
    if composite_cfg.get("type", "BASIC") != "BASIC":
        raise NotImplementedError("only the BASIC composite controller is implemented")
    arm = composite_cfg["body_parts"]["arms"]["right"]
    if arm["type"] not in ("OSC_POSE", "OSC_POSITION", "JOINT_VELOCITY", "JOINT_POSITION", "JOINT_TORQUE"):
        raise NotImplementedError(f"arm controller type {arm['type']} not implemented in the fused path")
    if arm["type"] in IMPEDANCE_KINDS and arm.get("impedance_mode", "fixed") not in IMPEDANCE_MODES:
        # the reference asserts the same at construction (osc.py, joint_pos.py: `impedance_mode in IMPEDANCE_MODES`)
        raise ValueError(f"{arm['type']}: unsupported impedance mode {arm.get('impedance_mode')!r}, not one of {sorted(IMPEDANCE_MODES)}")
    if arm["type"] == "JOINT_POSITION" and (arm.get("input_type", "delta") != "delta" or arm.get("qpos_limits") is not None):
        raise NotImplementedError("JOINT_POSITION: delta inputs, no qpos_limits")
    if arm["type"] == "JOINT_TORQUE" and arm.get("torque_limits") is not None:
        raise NotImplementedError("JOINT_TORQUE: torque_limits other than the actuator limits are not implemented")
    if arm["type"] in ("OSC_POSE", "OSC_POSITION") and (arm.get("input_type", "delta") != "delta"
                                                        or arm.get("input_ref_frame", "base") != "base" or arm.get("interpolation") is not None):
        raise NotImplementedError("fused OSC path implements delta inputs in the base frame")
    if arm.get("interpolation") is not None:
        raise NotImplementedError("interpolators are not implemented")
    if arm["type"] in ("OSC_POSE", "OSC_POSITION"):
        # the reference itself raises NotImplementedError when a goal would have to be clipped (osc.py:345-347 `position_limits`,
        # :398-400 `orientation_limits`): same behaviour, at configuration time instead of at the first set_goal
        if arm.get("position_limits") is not None:
            raise NotImplementedError("OSC position_limits: not implemented (the reference raises in compute_goal_pos, osc.py:345-347)")
        if arm.get("orientation_limits") is not None and np.array(arm.get("orientation_limits")).any():
            raise NotImplementedError("OSC orientation_limits: not implemented (the reference raises in compute_goal_ori, osc.py:398-400)")
    jn, an, sn = model.names["joint"], model.names["actuator"], model.names["site"]
    # arm joints: the robot's own hinge joints (robots/robot.py:302-332 collects them through the robot model)
    arm_j = [i for i, n in enumerate(jn) if n and n.startswith(robot_prefix) and int(model.jnt_type[i]) == 3]
    c = cfg_struct_cls()
    # kind 5 = OSC_POSITION (3-dim arm action; the orientation goal is re-anchored at every policy step)
    c.kind = {"OSC_POSE": 1, "JOINT_VELOCITY": 2, "JOINT_POSITION": 3, "JOINT_TORQUE": 4, "OSC_POSITION": 5}[arm["type"]]
    c.n_arm = len(arm_j)
    for k, j in enumerate(arm_j):
        c.arm_dof[k] = int(model.jnt_dofadr[j])
        c.arm_qpos[k] = int(model.jnt_qposadr[j])
        c.arm_act[k] = [i for i in range(model.nu) if model.actuator_trnid[i] == j][0]
    c.eef_site = sn.index(gripper_prefix + "grip_site")
    c.base_site = sn.index(robot_prefix + "right_center")
    grip_act = [i for i, n in enumerate(an) if n and n.startswith(gripper_prefix.replace("_right_", "_right_gripper_"))]
    if not grip_act:
        grip_act = [i for i, n in enumerate(an) if n and n.startswith("gripper0_")]
    c.n_grip = len(grip_act)
    for k, a in enumerate(grip_act):
        c.grip_act[k] = a
        c.grip_sign[k] = GRIPPER_SIGNS[gripper][k]
    c.grip_speed = GRIPPER_SPEED[gripper]
    if arm["type"] in ("JOINT_POSITION", "JOINT_TORQUE"):
        # per-joint scaling in the jv_in/out fields, gains in jv_kp / jv_kd (joint_pos.py:124-137: kd = 2 sqrt(kp) damping_ratio)
        n = c.n_arm
        c.action_dim = n + 1
        imax, imin = _arr(arm.get("input_max", 1), n), _arr(arm.get("input_min", -1), n)
        omax, omin = _arr(arm.get("output_max", 0.05), n), _arr(arm.get("output_min", -0.05), n)
        kp = _arr(arm.get("kp", 50), n)
        kd = _arr(arm["kd"], n) if arm.get("kd") is not None else 2 * np.sqrt(kp) * _arr(arm.get("damping_ratio", 1), n)
        for k in range(n):
            c.jv_kp[k], c.jv_ki[k], c.jv_kd[k] = kp[k], 0.0, kd[k]
            c.jv_in_max[k], c.jv_in_min[k], c.jv_out_max[k], c.jv_out_min[k] = imax[k], imin[k], omax[k], omin[k]
        c.jv_torque_comp = int(bool(arm.get("use_torque_compensation", True)))
        c.null_kp = 10.0
        c.uncouple_pos_ori = 1
        c.n_obs_site = 0
        if arm["type"] == "JOINT_POSITION":
            _impedance(c, arm, n, n)
        return c
    if arm["type"] == "JOINT_VELOCITY":
        n = c.n_arm
        c.action_dim = n + 1
        lo = np.array([model.actuator_ctrlrange[c.arm_act[k], 0] for k in range(n)])
        hi = np.array([model.actuator_ctrlrange[c.arm_act[k], 1] for k in range(n)])
        kp_in = arm.get("kp", 0.25)
        kp = kp_in * (hi - lo) if isinstance(kp_in, (int, float)) else _arr(kp_in, n)  # joint_vel.py:97-103
        imax, imin = _arr(arm.get("input_max", 1), n), _arr(arm.get("input_min", -1), n)
        omax, omin = _arr(arm.get("output_max", 1), n), _arr(arm.get("output_min", -1), n)
        for k in range(n):
            c.jv_kp[k], c.jv_ki[k], c.jv_kd[k] = kp[k], kp[k] * 0.005, kp[k] * 0.001
            c.jv_in_max[k], c.jv_in_min[k], c.jv_out_max[k], c.jv_out_min[k] = imax[k], imin[k], omax[k], omin[k]
        vl = arm.get("velocity_limits")
        c.jv_use_vel_limits = int(vl is not None)
        if vl is not None:
            c.jv_vel_lo, c.jv_vel_hi = float(vl[0]), float(vl[1])
        c.jv_torque_comp = int(bool(arm.get("use_torque_compensation", True)))
        c.null_kp = 10.0
        c.uncouple_pos_ori = 1
        c.n_obs_site = 0
        return c
    od = 3 if arm["type"] == "OSC_POSITION" else 6
    kp, dr = _arr6(arm["kp"]), _arr6(arm["damping_ratio"])

    def _lim(v):  # OSC_POSITION carries 3-vectors (osc.py:165): pad the unused orientation slots
        a = np.asarray(v, dtype=np.float64)
        return _arr6(v) if a.ndim == 0 or a.size == 6 else np.concatenate([a, np.ones(6 - a.size) * a.flat[0]])

    imax, imin = _lim(arm["input_max"]), _lim(arm["input_min"])
    omax, omin = _lim(arm["output_max"]), _lim(arm["output_min"])
    for k in range(6):
        c.kp[k], c.damping_ratio[k] = kp[k], dr[k]
        c.input_max[k], c.input_min[k], c.output_max[k], c.output_min[k] = imax[k], imin[k], omax[k], omin[k]
    c.null_kp = 10.0
    c.uncouple_pos_ori = int(bool(arm.get("uncouple_pos_ori", True)))
    c.n_obs_site = 0
    _impedance(c, arm, 6, od)
    return c
