"""OverrideOracleSim with the joint and contact fields and the device perturbation: the CPU counterpart of
BatchedSim.model_override (all nine fields), perturb_config and perturb_model for the tests.  perturb_model runs the numpy
restatement of the device draws (tests/dynamics_override_host.py); each environment's oracle is rebuilt from a host model with its
own values at set_const and at masked resets, as in the parent class."""
import numpy as np
import torch

from oracle.pyoracle import Oracle
from robosuite_b200.engine import DOF_FIELDS, PERTURB_SCALE, PERTURB_SHIFT, B2SError, normalize_perturb_spec
from robosuite_b200.mjcf.compiler import pack_model
from tests.dynamics_override_host import ALL_FIELDS, dynamics_invalid, dynamics_override_model, perturb_values
from tests.oracle_sim_override import OverrideOracleSim


class DynamicsOracleSim(OverrideOracleSim):
    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self._pert = []
        self.perturb_calls = []  # (mask, seed, counter) of every perturb_model call, for the tests

    def model_override(self, field, obj_id=None):
        if field not in ALL_FIELDS:
            raise B2SError("unknown field " + field)
        if field in DOF_FIELDS:
            if obj_id not in (None, -1):
                raise B2SError("the dof fields are whole vectors (id -1)")
            key = (field, -1)
            if key not in self._mov:
                self._mov[key] = torch.as_tensor(np.tile(np.asarray(getattr(self.model, field), dtype=np.float64), (self.n_env, 1)))
            return self._mov[key]
        return super().model_override(field, obj_id)

    def _set_const_env(self, e):
        vals = {}
        for (field, i), t in self._mov.items():
            vals.setdefault(field, {})[i] = t[e].numpy().copy()
        old, o = self.o[e], Oracle(pack_model(dynamics_override_model(self.model, **vals)))
        if self._cfg is not None:
            o.ctrl_setup(self._cfg)
            o.ctrl_state = old.ctrl_state
        self.o[e] = o
        return 128 if dynamics_invalid(self.model, **vals) else 0

    def perturb_config(self, spec):
        entries = normalize_perturb_spec(spec)
        for f, i, mode, amp, _ in entries:
            key = (f, -1) if f in DOF_FIELDS else (f, i)
            if key not in self._mov or mode not in (PERTURB_SCALE, PERTURB_SHIFT) or not (np.isfinite(amp) and amp >= 0) \
                    or (mode == PERTURB_SCALE and amp >= 1):
                raise B2SError("bad perturbation entry %r" % ((f, i, mode, amp),))
        self._pert = entries

    def perturb_model(self, mask=None, seed=0, counter=0):
        self.perturb_calls.append((None if mask is None else mask.clone(), seed, counter))
        if not self._pert:
            return
        envs = [e for e in range(self.n_env) if mask is None or bool(mask[e])]
        vals = perturb_values(self.model, self._pert, envs, seed, counter)
        for k, (f, i, *_) in enumerate(self._pert):
            t = self._mov[(f, -1) if f in DOF_FIELDS else (f, i)]
            v = torch.as_tensor(vals[k], dtype=t.dtype)
            idx = torch.as_tensor(envs, dtype=torch.long)
            if f in DOF_FIELDS and i >= 0:
                t[idx, i] = v[:, 0]
            elif t.ndim == 1:
                t[idx] = v[:, 0]
            else:
                t[idx] = v
