"""OracleSim with the per-environment object selection: the CPU counterpart of BatchedSim.obs_objects and the OB_SEL_* table ops
for the tests.  Environment e's selected rows read body body_ids[obj_sel[e]] of its oracle; a selection outside the list gives 0
and warn bit 512, as on the device."""
import torch

from robosuite_b200.envs.base import OB_SEL_BODY_POS, OB_SEL_BODY_QUAT_XYZW, OB_SEL_INDEX
from tests.oracle_sim import OracleSim


class SelectOracleSim(OracleSim):
    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self._sel_bodies, self.obj_sel, self._env = [], None, None

    def obs_objects(self, body_ids):
        self._sel_bodies = [int(b) for b in body_ids]
        if not self._sel_bodies:
            self.obj_sel = None
            return None
        if self.obj_sel is None:
            self.obj_sel = torch.zeros(self.n_env, dtype=torch.int32)
        return self.obj_sel

    def _value(self, o, op, a, b, prev, fresh):
        if op not in (OB_SEL_BODY_POS, OB_SEL_BODY_QUAT_XYZW, OB_SEL_INDEX):
            return super()._value(o, op, a, b, prev, fresh)
        k = int(self.obj_sel[self._env])
        if not 0 <= k < len(self._sel_bodies):
            self.warn[self._env] |= 512
            return 0.0
        body = self._sel_bodies[k]
        if op == OB_SEL_INDEX:
            return float(k)
        return o.xpos[body][b] if op == OB_SEL_BODY_POS else o.xquat[body][(b + 1) & 3]

    def _sample_obs(self, e):
        self._env = e
        super()._sample_obs(e)

    def _sample_task(self, e):
        self._env = e
        super()._sample_task(e)
