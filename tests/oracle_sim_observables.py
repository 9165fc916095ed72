"""OracleSim with observable sampling rates and corruptors: the CPU counterpart of BatchedSim.obs_modifiers for the tests.

env_step runs the substeps one by one (step1 -> controller (the action on the first substep) -> step2, what o_env_step does) and
after each one advances the timers of tests/observable_ref.py; an observable that is due samples its rows from this substep's state
and corrupts them with the numpy restatement of the device draws.  Without modifiers the observation is sampled after the last
substep, as in OracleSim."""
import numpy as np
import torch

from tests.observable_ref import check_modifiers, corrupt, obs_update, quat2mat
from tests.oracle_sim import OB_REL_QUAT_LAG, OracleSim, _m2q_xyzw_wpos, _q2m


class ObsOracleSim(OracleSim):
    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self._mods = None  # (row_obs, mods, seed) while configured
        self.obs_timer = self.obs_sampled = self.obs_nsample = None

    def obs_modifiers(self, row_obs, mods, seed=0):
        mods = [tuple(float(x) if i != 1 else int(x) for i, x in enumerate(m)) for m in mods]
        if self._obs_tab is None:
            from robosuite_b200.engine import B2SError

            raise B2SError("b2s_obs_modifiers: observations are not configured")
        check_modifiers(len(self._obs_tab[0]), row_obs, mods)
        if not mods:
            self._mods = None
            return
        n = len(mods)
        if self.obs_timer is None or self.obs_timer.shape[1] != n:
            self.obs_timer = torch.zeros((self.n_env, n), dtype=torch.float64)
            self.obs_sampled = torch.zeros(self.n_env, dtype=torch.int32)
            self.obs_nsample = torch.zeros((self.n_env, n), dtype=torch.int32)
            self._mods = None
        if self._mods is None:  # the default rule's state at a control-step boundary
            self.obs_timer[:] = float(self.model.opt_timestep)
            self.obs_sampled[:] = (1 << n) - 1 if n < 32 else -1
        self._mods = (np.asarray(row_obs, dtype=np.int64).copy(), mods, int(seed) & (2 ** 64 - 1))

    def _value(self, o, op, a, b, prev, fresh):
        """with modifiers the cached quaternion of a lagged entry may be corrupted: the reference's quat2mat normalises it"""
        if op != OB_REL_QUAT_LAG or self._mods is None or fresh or prev is None:
            return super()._value(o, op, a, b, prev, fresh)
        qs, comp, body = a >> 12, b & 255, (b >> 16) & 255
        return _m2q_xyzw_wpos(_q2m(o.xquat[body]).T @ quat2mat(prev[qs:qs + 4]))[comp]

    def _due(self, e, force):
        """advance environment e's timers by one substep (force: reset()'s update from t = 0); bit o = observable o samples"""
        _, mods, _ = self._mods
        dt = float(self.model.opt_timestep)
        bits, due = int(self.obs_sampled[e]) & 0xFFFFFFFF, 0
        for o, m in enumerate(mods):
            t, s = (0.0, False) if force else (float(self.obs_timer[e, o]), bool((bits >> o) & 1))
            t, s, take = obs_update(t, s, m[0], dt, force=force)
            self.obs_timer[e, o] = t
            bits = (bits | (1 << o)) if s else (bits & ~(1 << o))
            due |= int(take) << o
        self.obs_sampled[e] = bits if bits < 2 ** 31 else bits - 2 ** 32
        return due

    def _sample_obs(self, e, due=None):
        if self._mods is None or self._obs_tab is None:
            return super()._sample_obs(e)
        if due is None:  # forward of a fresh environment / reset: the forced update
            due = self._due(e, True)
        if not due:
            return
        row_obs, mods, seed = self._mods
        o, prev, fresh = self.o[e], self.obs[e].numpy().copy(), bool(self.obs_fresh[e])
        op, a, b = self._obs_tab
        for ob, m in enumerate(mods):
            if not (due >> ob) & 1:
                continue
            rows = np.nonzero(row_obs[:len(op)] == ob)[0]
            vals = [self._value(o, int(op[k]), int(a[k]), int(b[k]), prev, fresh) for k in rows]
            self.obs[e, rows] = torch.as_tensor(corrupt(vals, m, seed, e, int(self.obs_nsample[e, ob]), rows))
            self.obs_nsample[e, ob] += 1
        self.obs_fresh[e] = 0

    def env_step(self, action, n_substeps):
        act = action.numpy().astype(np.float64)
        for e in range(self.n_env):
            self._push(e)
            oe = self.o[e]
            for sub in range(n_substeps):
                oe.step1()
                oe.ctrl_run(act[e] if sub == 0 else None)
                oe.step2()
                if self._mods is not None and self._obs_tab is not None:
                    self._sample_obs(e, self._due(e, False))
            self._pull(e)
            if self._mods is None:
                self._sample_obs(e)  # last substep: poses of its step1, qpos / qvel after its step2
            self._sample_task(e)
