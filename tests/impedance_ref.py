"""Variable impedance (impedance_mode "variable" / "variable_kp" of OSC_POSE, OSC_POSITION and JOINT_POSITION) for tests only: the
gain part of the action over the fp64 restatement of tests/controller_ref.py, and a CPU stand-in that runs the unchanged oracle in
these modes.

Reference semantics, recalled from robosuite v1.5 controllers/parts/arm/osc.py and parts/generic/joint_pos.py set_goal (no
reference checkout was available to check them against), with d = 6 for both OSC kinds and n_arm for JOINT_POSITION:
  "variable"     action = [damping_ratio (d), kp (d), delta, gripper]:  kp = clip(kp, kp_min, kp_max),
                                                                        kd = 2 sqrt(kp) clip(damping_ratio, dr_min, dr_max)
  "variable_kp"  action = [kp (d), delta, gripper]:                     kp = clip(kp, kp_min, kp_max), kd = 2 sqrt(kp)
The gains are set on the policy substep before the goal and hold until the next one; a reset restores the configured gains.  A
gain row is kp[8], kd[8] (the device's "ctrl_gain" layout)."""
import types

import numpy as np
import torch

from tests import controller_ref as ref
from tests.oracle_sim import OracleSim

FIXED, VARIABLE, VARIABLE_KP = 0, 1, 2
MODE_NAMES = {"variable": VARIABLE, "variable_kp": VARIABLE_KP}


def gain_dim(cfg):
    return cfg.n_arm if cfg.kind == 3 else 6


def delta_offset(cfg):
    """where the delta starts in the action"""
    return {FIXED: 0, VARIABLE_KP: 1, VARIABLE: 2}[int(cfg.impedance_mode)] * gain_dim(cfg)


def configured_gains(cfg):
    """the gain row of the configured (fixed) gains"""
    row, d = np.zeros(16), gain_dim(cfg)
    if cfg.kind == 3:
        row[:d], row[8:8 + d] = list(cfg.jv_kp)[:d], list(cfg.jv_kd)[:d]
    else:
        kp = np.array(list(cfg.kp)[:6])
        row[:6], row[8:14] = kp, 2.0 * np.sqrt(kp) * np.array(list(cfg.damping_ratio)[:6])
    return row


def gains_from_action(cfg, action):
    """the gain row set_goal makes from one environment's action"""
    a, d, row = np.asarray(action, dtype=np.float64), gain_dim(cfg), np.zeros(16)
    lim = {f: np.array(list(getattr(cfg, f))[:d]) for f in ("kp_min", "kp_max", "damping_ratio_min", "damping_ratio_max")}
    if int(cfg.impedance_mode) == VARIABLE:
        kp = np.clip(a[d:2 * d], lim["kp_min"], lim["kp_max"])
        kd = 2.0 * np.sqrt(kp) * np.clip(a[:d], lim["damping_ratio_min"], lim["damping_ratio_max"])
    else:
        kp = np.clip(a[:d], lim["kp_min"], lim["kp_max"])
        kd = 2.0 * np.sqrt(kp)
    row[:d], row[8:8 + d] = kp, kd
    return row


def fixed_view(cfg, gain):
    """a fixed-mode copy of `cfg` (every field, as plain lists) whose gains are the row `gain`: what controller_ref runs.  The OSC
    restatement forms kd = 2 sqrt(kp) damping_ratio itself, so the view carries damping_ratio = kd / (2 sqrt(kp)) (0 where kp = 0:
    kd is 0 there), which returns kd to within rounding"""
    v = types.SimpleNamespace(**{f: (list(getattr(cfg, f)) if hasattr(getattr(cfg, f), "__len__") else getattr(cfg, f))
                                 for f, _ in type(cfg)._fields_})
    d = gain_dim(cfg)
    v.action_dim = cfg.action_dim - delta_offset(cfg)
    v.impedance_mode = FIXED
    if cfg.kind == 3:
        v.jv_kp[:d], v.jv_kd[:d] = list(gain[:d]), list(gain[8:8 + d])
    else:
        kp, kd = np.asarray(gain[:6]), np.asarray(gain[8:14])
        v.kp = list(kp)
        v.damping_ratio = list(np.where(kp > 0, kd / (2.0 * np.sqrt(np.where(kp > 0, kp, 1.0))), 0.0))
    return v


def run(model, cfg, inp, state, gain, action=None, goal_ori=None):
    """controller_ref.run (or run_given_goal with `goal_ori`) in a variable mode: on a policy substep the gains come from the
    action, then the fixed controller runs on the delta part with them.  `gain`: the row at the start of the substep.  Returns
    run's dict with the new row under "gain"."""
    if action is not None:
        gain = gains_from_action(cfg, action)
        action = np.asarray(action, dtype=np.float64)[delta_offset(cfg):]
    v = fixed_view(cfg, gain)
    r = ref.run(model, v, inp, state, action) if goal_ori is None else ref.run_given_goal(model, v, inp, state, action, goal_ori)
    r["gain"] = np.asarray(gain, dtype=np.float64).copy()
    return r


def gain_action(cfg, gain_row, delta_action):
    """the variable-mode action that sets the gains of `gain_row` (damping ratio = kd / (2 sqrt(kp)), 1 where kp = 0) and then
    takes the fixed-mode action `delta_action`"""
    d = gain_dim(cfg)
    kp, kd = np.asarray(gain_row[:d]), np.asarray(gain_row[8:8 + d])
    parts = [kp, np.asarray(delta_action, dtype=np.float64)]
    if int(cfg.impedance_mode) == VARIABLE:
        parts.insert(0, np.where(kp > 0, kd / (2.0 * np.sqrt(np.where(kp > 0, kp, 1.0))), 1.0))
    return np.concatenate(parts)


class ImpedanceOracleSim(OracleSim):
    """OracleSim in the variable modes, with the oracle itself unchanged: each environment's oracle gets its own copy of the
    fixed-mode configuration, whose gains are set from the action before every step (OSC: kp and damping_ratio, from which the
    oracle forms kd = 2 sqrt(kp) damping_ratio as the device does; JOINT_POSITION: jv_kp and jv_kd), and is stepped with the delta
    part.  Resets restore the configured gains.  `ctrl_gain` mirrors the device's array."""

    def ctrl_config(self, cfg):
        super().ctrl_config(cfg)
        self._icfg = cfg
        self._mode = int(getattr(cfg, "impedance_mode", FIXED))
        if self._mode == FIXED:
            return
        self._cfg.action_dim = cfg.action_dim - delta_offset(cfg)
        self._ecfg = []
        for o in self.o:
            c = type(self._cfg).from_buffer_copy(self._cfg)
            self._ecfg.append(c)
            o.ctrl_cfg = c
        self.ctrl_gain = torch.as_tensor(np.tile(configured_gains(cfg), (self.n_env, 1)))
        for e in range(self.n_env):
            self._set_gains(e)

    def _set_gains(self, e):
        c, g, d = self._ecfg[e], self.ctrl_gain[e].numpy(), gain_dim(self._icfg)
        if self._icfg.kind == 3:
            c.jv_kp[:d], c.jv_kd[:d] = list(g[:d]), list(g[8:8 + d])
        else:  # kd = 2 sqrt(kp) dr in the oracle: the damping ratio that was clipped ("variable") or 1 ("variable_kp")
            c.kp[:6] = list(g[:6])

    def _reset_gains(self, mask):
        if getattr(self, "_mode", FIXED) == FIXED:
            return
        for e in range(self.n_env):
            if mask is None or bool(mask[e]):
                self.ctrl_gain[e] = torch.as_tensor(configured_gains(self._icfg))
                if self._icfg.kind != 3:
                    self._ecfg[e].damping_ratio[:6] = list(self._icfg.damping_ratio)[:6]
                self._set_gains(e)

    def reset_envs(self, mask=None, qpos=None):
        super().reset_envs(mask, qpos)
        self._reset_gains(mask)

    def ctrl_reset(self, mask=None):
        super().ctrl_reset(mask)
        self._reset_gains(mask)

    def env_step(self, action, n_substeps):
        if self._mode == FIXED:
            return super().env_step(action, n_substeps)
        act = action.numpy().astype(np.float64)
        cfg, d = self._icfg, gain_dim(self._icfg)
        for e in range(self.n_env):
            self.ctrl_gain[e] = torch.as_tensor(gains_from_action(cfg, act[e]))
            if cfg.kind != 3:
                dr = (np.clip(act[e, :d], list(cfg.damping_ratio_min)[:d], list(cfg.damping_ratio_max)[:d])
                      if self._mode == VARIABLE else np.ones(d))
                self._ecfg[e].damping_ratio[:6] = list(dr)
            self._set_gains(e)
        return super().env_step(torch.as_tensor(act[:, delta_offset(cfg):]), n_substeps)
