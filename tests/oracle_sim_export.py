"""OracleSim with the array-group exports: the CPU counterpart of BatchedSim's set_contact_export / set_step1_export /
set_step2_export / set_export, contacts() and `data` for the tests.  The rule is the device's: after every env_step a group is
written when the full export or the group's own export is on, and forward / reset_envs write every group for their environments.
Environment e's rows are then its oracle's arrays of the last substep as the device writes them:
  - the contact records: data.contact[:ncon] in order (ncon, contact_geom / dim / dist / pos / frame / friction), rows
    ncon .. maxcon - 1 geom -1 and zeros;
  - the step-1 arrays: poses of the colliding geoms only (the others stay zero), the dense mass matrix;
  - the step-2 arrays: the row arrays at capacity with zeros from row nefc on (efc_J keeps its earlier values there), and
    contact_efc_address, the oracle's data.contact[c].efc_address with -1 from ncon on.
The Jacobians come from the oracle's own mj_jac at the exported points, not from the exported cdof."""
import numpy as np
import torch

from robosuite_b200.data import BatchedData
from tests.oracle_sim import OracleSim

STEP1 = ("xpos", "xquat", "xmat", "site_xpos", "site_xmat", "cdof", "qfrc_bias", "qfrc_passive")
STEP2_NV = ("qfrc_actuator", "qfrc_smooth", "qacc_smooth", "qfrc_constraint")


class ExportOracleSim(OracleSim):
    def __init__(self, model, n_env, device=0, precision="f64", maxcon=None, maxefc=None, tier_small=None):
        super().__init__(model, n_env, device, precision, maxcon, maxefc, tier_small)
        mc = int(maxcon or getattr(model, "opt_maxcon", None) or 32)
        me = int(maxefc or getattr(model, "opt_maxefc", None) or 64)
        nb, ns, ng, nv, nu = model.nbody, model.nsite, model.ngeom, model.nv, model.nu
        z = lambda *s: torch.zeros(s, dtype=torch.float64)
        zi = lambda *s: torch.zeros(s, dtype=torch.int32)
        # contact records
        self.ncon, self.contact_dim = zi(n_env), zi(n_env, mc)
        self.contact_geom = torch.full((n_env, mc, 2), -1, dtype=torch.int32)
        self.contact_dist, self.contact_pos, self.contact_frame = z(n_env, mc), z(n_env, mc, 3), z(n_env, mc, 9)
        self.contact_friction = z(n_env, mc, 3)
        # step-1 arrays
        self.xpos, self.xquat, self.xmat = z(n_env, nb, 3), z(n_env, nb, 4), z(n_env, nb, 9)
        self.site_xpos, self.site_xmat = z(n_env, ns, 3), z(n_env, ns, 9)
        self.geom_xpos, self.geom_xmat = z(n_env, ng, 3), z(n_env, ng, 9)
        self.qM, self.cdof, self.qfrc_bias, self.qfrc_passive = z(n_env, nv, nv), z(n_env, nv, 6), z(n_env, nv), z(n_env, nv)
        self._cg = sorted({int(g) for p in model.pair_geom for g in p})
        # step-2 arrays
        for name in STEP2_NV:
            setattr(self, name, z(n_env, nv))
        self.actuator_force = z(n_env, nu)
        self.nefc, self.solver_niter = zi(n_env), zi(n_env)
        self.efc_type = zi(n_env, me)
        self.efc_D, self.efc_R, self.efc_aref, self.efc_force = z(n_env, me), z(n_env, me), z(n_env, me), z(n_env, me)
        self.efc_J = z(n_env, me, nv)
        self.contact_efc_address = torch.full((n_env, mc), -1, dtype=torch.int32)
        self.full_export, self.contact_export, self.step1_export, self.step2_export = True, False, False, False
        self.data = BatchedData(self)

    def set_export(self, flag):
        self.full_export = bool(flag)

    def set_contact_export(self, flag):
        self.contact_export = bool(flag)

    def set_step1_export(self, flag):
        self.step1_export = bool(flag)

    def set_step2_export(self, flag):
        self.step2_export = bool(flag)

    def contacts(self):
        return {"ncon": self.ncon, "geom": self.contact_geom, "dist": self.contact_dist, "pos": self.contact_pos,
                "frame": self.contact_frame, "friction": self.contact_friction}

    def _export_contacts(self, e):
        cons = self.o[e].contacts()[: self.contact_geom.shape[1]]
        self.ncon[e] = len(cons)
        self.contact_geom[e] = -1
        for t in (self.contact_dim, self.contact_dist, self.contact_pos, self.contact_frame, self.contact_friction):
            t[e] = 0
        for k, c in enumerate(cons):
            self.contact_geom[e, k] = torch.tensor([c["geom1"], c["geom2"]], dtype=torch.int32)
            self.contact_dim[e, k] = int(c["dim"])
            self.contact_dist[e, k] = float(c["dist"])
            self.contact_pos[e, k] = torch.as_tensor(np.asarray(c["pos"]))
            self.contact_frame[e, k] = torch.as_tensor(np.asarray(c["frame"]).reshape(9))
            self.contact_friction[e, k] = torch.as_tensor(np.asarray(c["friction"])[[0, 2, 3]])  # (slide, spin, roll)

    def _export_step1(self, e):
        o = self.o[e]
        for name in STEP1:
            getattr(self, name)[e] = torch.as_tensor(getattr(o, name).copy())
        self.qM[e] = torch.as_tensor(o.M.copy())
        self.geom_xpos[e, self._cg] = torch.as_tensor(o.geom_xpos[self._cg].copy())
        self.geom_xmat[e, self._cg] = torch.as_tensor(o.geom_xmat[self._cg].copy())

    def _export_step2(self, e):
        o = self.o[e]
        for name in STEP2_NV + ("actuator_force",):
            getattr(self, name)[e] = torch.as_tensor(getattr(o, name).copy())
        me = self.efc_force.shape[1]
        n = min(int(o.nefc), me)
        self.nefc[e], self.solver_niter[e] = n, int(o.geti("solver_niter"))
        for name in ("type", "D", "R", "aref", "force"):
            t = getattr(self, "efc_" + name)
            t[e] = 0
            t[e, :n] = torch.as_tensor(np.asarray(o.efc(name))[:n].copy()).to(t.dtype)
        self.efc_J[e, :n] = torch.as_tensor(o.efc("J")[:n].copy())
        self.contact_efc_address[e] = -1
        for k, c in enumerate(o.contacts()[: self.contact_efc_address.shape[1]]):
            self.contact_efc_address[e, k] = int(c["efc_address"])

    def _sample_task(self, e):
        # runs after every step, forward and reset of environment e, on the arrays of its last substep
        super()._sample_task(e)
        every = self.full_export or self._forwarding
        if every or self.contact_export:
            self._export_contacts(e)
        if every or self.step1_export:
            self._export_step1(e)
        if every or self.step2_export:
            self._export_step2(e)

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
