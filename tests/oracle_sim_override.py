"""OracleSim with per-environment model values: the CPU counterpart of BatchedSim.model_override / set_const for the tests.  The
oracle of an environment is rebuilt from a host copy of the model with that environment's override values
(tests/model_override_host.py) whenever the engine would run its set-constants pass: set_const() and the masked reset."""
import numpy as np
import torch

from oracle.pyoracle import Oracle
from robosuite_b200.mjcf.compiler import pack_model
from tests.model_override_host import invalid, override_model
from tests.oracle_sim import OracleSim


class OverrideOracleSim(OracleSim):
    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self._mov = {}  # (field, object id) -> [n_env, ...] values

    def model_override(self, field, obj_id):
        """same surface as BatchedSim.model_override: per-environment values, initialised to the model's"""
        key = (field, int(obj_id))
        if key not in self._mov:
            v = np.asarray(getattr(self.model, field)[int(obj_id)], dtype=np.float64)
            self._mov[key] = torch.as_tensor(np.tile(v, (self.n_env, 1)) if v.ndim else np.full(self.n_env, float(v)))
        return self._mov[key]

    def _set_const_env(self, e):
        """rebuild environment e's oracle from a host model with its override values; returns warn bit 128 for invalid values"""
        vals = {}
        for (field, i), t in self._mov.items():
            vals.setdefault(field, {})[i] = t[e].numpy().copy()
        old, o = self.o[e], Oracle(pack_model(override_model(self.model, **vals)))
        if self._cfg is not None:
            o.ctrl_setup(self._cfg)
            o.ctrl_state = old.ctrl_state
        self.o[e] = o
        return 128 if invalid(self.model, **vals) else 0

    def _masked(self, mask):
        return [e for e in range(self.n_env) if mask is None or bool(mask[e])] if self._mov else []

    def set_const(self, mask=None):
        for e in self._masked(mask):
            self.warn[e] |= self._set_const_env(e)

    def reset_envs(self, mask=None, qpos=None):
        """b2s_reset_envs on a handle with overrides: the set-constants pass runs after the warn bits are cleared, before the forward"""
        bits = {e: self._set_const_env(e) for e in self._masked(mask)}
        super().reset_envs(mask, qpos)
        for e, b in bits.items():
            self.warn[e] |= b
