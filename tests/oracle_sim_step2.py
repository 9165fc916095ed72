"""DataOracleSim with the step-2 export and the contact records: the CPU counterpart of BatchedSim.set_step2_export /
set_contact_export and `data`'s step-2 half for the tests.  After every env_step (with the step-2 or the full export on) and for
the environments of every forward / reset_envs, environment e's rows are its oracle's arrays of the last substep as the device
writes them: the row arrays at capacity with zeros from row nefc on (efc_J keeps its earlier values there), and
contact_efc_address, the oracle's data.contact[c].efc_address with -1 from ncon on.  The contact records follow the contact
export's rule (ncon, contact_geom / dim / dist / pos / frame / friction, rows ncon .. maxcon - 1 geom -1 and zeros)."""
import numpy as np
import torch

from tests.oracle_sim_data import DataOracleSim

STEP2_NV = ("qfrc_actuator", "qfrc_smooth", "qacc_smooth", "qfrc_constraint")


class Step2OracleSim(DataOracleSim):
    def __init__(self, model, n_env, device=0, precision="f64", maxcon=None, maxefc=None, tier_small=None):
        super().__init__(model, n_env, device, precision, maxcon, maxefc, tier_small)
        mc = int(maxcon or getattr(model, "opt_maxcon", None) or 32)
        me = int(maxefc or getattr(model, "opt_maxefc", None) or 64)
        nv, nu = model.nv, model.nu
        z = lambda *s: torch.zeros(s, dtype=torch.float64)
        zi = lambda *s: torch.zeros(s, dtype=torch.int32)
        for name in STEP2_NV:
            setattr(self, name, z(n_env, nv))
        self.actuator_force = z(n_env, nu)
        self.nefc, self.solver_niter, self.ncon = zi(n_env), zi(n_env), zi(n_env)
        self.efc_type = zi(n_env, me)
        self.efc_D, self.efc_R, self.efc_aref, self.efc_force = z(n_env, me), z(n_env, me), z(n_env, me), z(n_env, me)
        self.efc_J = z(n_env, me, nv)
        self.contact_efc_address = torch.full((n_env, mc), -1, dtype=torch.int32)
        self.contact_geom = torch.full((n_env, mc, 2), -1, dtype=torch.int32)
        self.contact_dim = zi(n_env, mc)
        self.contact_dist, self.contact_pos, self.contact_frame = z(n_env, mc), z(n_env, mc, 3), z(n_env, mc, 9)
        self.contact_friction = z(n_env, mc, 3)
        self.step2_export = self.contact_export = False

    def set_step2_export(self, flag):
        self.step2_export = bool(flag)

    def set_contact_export(self, flag):
        self.contact_export = bool(flag)

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

    def _sample_task(self, e):
        # runs after every step, forward and reset of environment e, on the arrays of its last substep
        super()._sample_task(e)
        if self.full_export or self.step2_export or self._forwarding:
            self._export_step2(e)
        if self.full_export or self.contact_export or self._forwarding:
            self._export_contacts(e)
