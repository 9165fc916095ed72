"""OracleSim with the contact export: the CPU counterpart of BatchedSim.set_contact_export / contacts() for the tests.  After
every env_step (with the export on) and for the environments of every forward / reset_envs, environment e's rows are its oracle's
data.contact[:ncon] in order, rows ncon .. maxcon - 1 geom -1 and zeros, as the device writes them."""
import numpy as np
import torch

from tests.oracle_sim import OracleSim


class ContactOracleSim(OracleSim):
    def __init__(self, model, n_env, device=0, precision="f64", maxcon=None, maxefc=None, tier_small=None):
        super().__init__(model, n_env, device, precision, maxcon, maxefc, tier_small)
        mc = int(maxcon or getattr(model, "opt_maxcon", None) or 32)
        z = lambda *s: torch.zeros(s, dtype=torch.float64)
        self.ncon = torch.zeros(n_env, dtype=torch.int32)
        self.contact_geom = torch.full((n_env, mc, 2), -1, dtype=torch.int32)
        self.contact_dist, self.contact_pos, self.contact_frame = z(n_env, mc), z(n_env, mc, 3), z(n_env, mc, 9)
        self.contact_friction = z(n_env, mc, 3)
        self._export_con = False

    def set_contact_export(self, flag):
        self._export_con = bool(flag)

    def contacts(self):
        return {"ncon": self.ncon, "geom": self.contact_geom, "dist": self.contact_dist, "pos": self.contact_pos,
                "frame": self.contact_frame, "friction": self.contact_friction}

    def _export(self, e):
        cons = self.o[e].contacts()[: self.contact_geom.shape[1]]
        self.ncon[e] = len(cons)
        self.contact_geom[e] = -1
        for t in (self.contact_dist, self.contact_pos, self.contact_frame, self.contact_friction):
            t[e] = 0
        for k, c in enumerate(cons):
            self.contact_geom[e, k] = torch.tensor([c["geom1"], c["geom2"]], dtype=torch.int32)
            self.contact_dist[e, k] = float(c["dist"])
            self.contact_pos[e, k] = torch.as_tensor(np.asarray(c["pos"]))
            self.contact_frame[e, k] = torch.as_tensor(np.asarray(c["frame"]).reshape(9))
            self.contact_friction[e, k] = torch.as_tensor(np.asarray(c["friction"])[[0, 2, 3]])  # (slide, spin, roll)

    def _sample_task(self, e):
        # runs after every step, forward and reset of environment e, on the contacts of its last step1
        super()._sample_task(e)
        if self._export_con or self._forwarding:
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
