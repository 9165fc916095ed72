"""SelectOracleSim with the placement program: the CPU counterpart of BatchedSim.place_config / place_objects for the tests.
place_objects runs the numpy restatement of the device's draws (tests/placement_ref.py) for the masked environments, writes the
free-joint rows of q and the pose overrides as the kernel does, and leaves warn bit 1024 pending for the next reset_envs."""
import numpy as np
import torch

from robosuite_b200.engine import B2SError
from tests.oracle_sim_select import SelectOracleSim
from tests.placement_ref import place_values


class PlacementOracleSim(SelectOracleSim):
    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self._prog, self._ov_local = [], {}
        self._pending = torch.zeros(self.n_env, dtype=torch.int32)
        self.place_calls = []  # (mask, seed, counter) of every place_objects call, for the tests

    def place_config(self, entries):
        m = self.model
        ov = getattr(self, "_ov", {})
        self._ov_local, self._ov_children = {}, {}
        for i, e in enumerate(entries):
            if (e["qpos_adr"] >= 0) == (e["body"] >= 0) or not -1 <= e["ref"] < i:
                raise B2SError("bad placement entry %d" % i)
            if e["body"] >= 0:
                if e["body"] not in ov:
                    raise B2SError("entry %d: the body has no pose override" % i)
                # the overridden bodies whose parent is the placed body (the models' only case: Door_frame under Door_main)
                self._ov_children[i] = [c for c in ov if c != e["body"] and int(m.body_parentid[c]) == e["body"]]
                self._ov_local[i] = [(np.asarray(m.body_pos[c], dtype=np.float64), np.asarray(m.body_quat[c], dtype=np.float64))
                                     for c in self._ov_children[i]]
        self._prog = list(entries)

    def place_objects(self, qpos, mask=None, seed=0, counter=0):
        self.place_calls.append((None if mask is None else mask.clone(), seed, counter))
        if not self._prog:
            return
        envs = [e for e in range(self.n_env) if mask is None or bool(mask[e])]
        q = qpos.numpy()  # a view: rows written in place
        res = place_values(self._prog, envs, seed, counter, qpos=q, ov_local=self._ov_local)
        for o, per_env in res["ov"].items():
            bodies = [self._prog[o]["body"]] + self._ov_children[o]
            for k, env in enumerate(envs):
                for b, (p, qq) in zip(bodies, per_env[k]):
                    P, Q, _ = self._ov[b]
                    P[env] = torch.as_tensor(np.asarray(p, dtype=np.float64))
                    Q[env] = torch.as_tensor(np.asarray(qq, dtype=np.float64))
        for k, env in enumerate(envs):
            self._pending[env] = int(res["warn"][k])

    def reset_envs(self, mask=None, qpos=None):
        super().reset_envs(mask, qpos)
        for e in range(self.n_env):
            if mask is None or bool(mask[e]):
                self.warn[e] = self._pending[e]
                self._pending[e] = 0
