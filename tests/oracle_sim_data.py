"""OracleSim with the step-1 export: the CPU counterpart of BatchedSim.set_step1_export / `data` for the tests.  After every
env_step (with the step-1 or the full export on) and for the environments of every forward / reset_envs, environment e's rows are its
oracle's step-1 arrays as the device writes them: poses of the colliding geoms only (the others stay zero), the dense mass matrix.
The Jacobians come from the oracle's own mj_jac at the exported points, not from the exported cdof."""
import numpy as np
import torch

from robosuite_b200.data import BatchedData
from tests.oracle_sim import OracleSim


class DataOracleSim(OracleSim):
    def __init__(self, model, n_env, device=0, precision="f64", maxcon=None, maxefc=None, tier_small=None):
        super().__init__(model, n_env, device, precision, maxcon, maxefc, tier_small)
        z = lambda *s: torch.zeros(s, dtype=torch.float64)
        nb, ns, ng, nv = model.nbody, model.nsite, model.ngeom, model.nv
        self.xpos, self.xquat, self.xmat = z(n_env, nb, 3), z(n_env, nb, 4), z(n_env, nb, 9)
        self.site_xpos, self.site_xmat = z(n_env, ns, 3), z(n_env, ns, 9)
        self.geom_xpos, self.geom_xmat = z(n_env, ng, 3), z(n_env, ng, 9)
        self.qM, self.cdof, self.qfrc_bias, self.qfrc_passive = z(n_env, nv, nv), z(n_env, nv, 6), z(n_env, nv), z(n_env, nv)
        self._cg = sorted({int(g) for p in model.pair_geom for g in p})
        self.full_export, self.step1_export = True, False
        self.data = BatchedData(self)

    def set_export(self, flag):
        self.full_export = bool(flag)

    def set_step1_export(self, flag):
        self.step1_export = bool(flag)

    def _export(self, e):
        o = self.o[e]
        for name in ("xpos", "xquat", "xmat", "site_xpos", "site_xmat", "cdof", "qfrc_bias", "qfrc_passive"):
            getattr(self, name)[e] = torch.as_tensor(getattr(o, name).copy())
        self.qM[e] = torch.as_tensor(o.M.copy())
        self.geom_xpos[e, self._cg] = torch.as_tensor(o.geom_xpos[self._cg].copy())
        self.geom_xmat[e, self._cg] = torch.as_tensor(o.geom_xmat[self._cg].copy())

    def _sample_task(self, e):
        # runs after every step, forward and reset of environment e, on the arrays of its last step1
        super()._sample_task(e)
        if self.full_export or self.step1_export or self._forwarding:
            self._export(e)

    _forwarding = False

    def forward(self):
        self._forwarding = True
        try:
            super().forward()
        finally:
            self._forwarding = False

    def reset_envs(self, mask=None, qpos=None):
        self._forwarding = True
        try:
            super().reset_envs(mask, qpos)
        finally:
            self._forwarding = False

    def full_m(self):
        return self.qM.clone()

    def _jac(self, points, bodies):
        jp = torch.zeros((self.n_env, 3, self.model.nv), dtype=torch.float64)
        jr = torch.zeros_like(jp)
        for e, o in enumerate(self.o):
            p, r = o.jac(points[e].numpy(), int(bodies))
            jp[e], jr[e] = torch.as_tensor(p), torch.as_tensor(r)
        return jp, jr

    def jac_body(self, body_id):
        return self._jac(self.xpos[:, body_id], body_id)

    def jac_site(self, site_id):
        return self._jac(self.site_xpos[:, site_id], np.asarray(self.model.site_bodyid)[site_id])

    def jac_geom(self, geom_id):
        return self._jac(self.geom_xpos[:, geom_id], np.asarray(self.model.geom_bodyid)[geom_id])
