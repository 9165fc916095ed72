"""Lift task (robosuite/environments/manipulation/lift.py) on the batched engine."""
import math

import numpy as np

from ..mjcf.compiler import quat2mat
from .base import (OB_BODY_MINUS_SITE, OB_BODY_POS, OB_BODY_QUAT_XYZW, BatchedMujocoEnv, load_task_model,
                   register_env)

PANDA_INIT_QPOS = np.array([0, np.pi / 16.0, 0.00, -np.pi / 2.0 - np.pi / 3.0, 0.00, np.pi - 0.2, np.pi / 4])
SAWYER_INIT_QPOS = np.array([0.00, -1.18, 0.00, 2.18, 0.00, 0.57, -1.57])
GRIPPER_INIT_QPOS = {"Panda": [0.020833, -0.020833], "Sawyer": [0.020833, -0.020833]}


@register_env
class BatchedLift(BatchedMujocoEnv):
    """suite.make("Lift", robots="Panda", num_envs=N): table arena + one cube, sparse/shaped lifting reward."""

    # capacities: the small tier holds every contact / row count seen in 10^5 random-action environment-substeps (max 12 / 47 observed,
    # mean 4 / 21); the large tier exists for the 1-in-10^6 pile-ups (an arm lying on the table next to the cube)
    maxcon, maxefc = 48, 128
    tier_small = (12, 44)

    table_offset = (0.0, 0.0, 0.8)  # lift.py:146
    cube_size_range = (0.020, 0.022)  # lift.py:311-314: half sizes of the cube, density 1000

    def __init__(self, *args, per_env_cube_size=False, **kwargs):
        """per_env_cube_size: every environment draws its own cube half sizes from U[0.020, 0.022]^3 (mass and moments from density
        1000), as the reference does per model build: at construction, and again at each of its resets when hard_reset=True.
        False: every environment keeps the cube of the model (the draw made when the fixture was compiled)."""
        if per_env_cube_size and kwargs.get("placement_initializer") is not None:
            raise NotImplementedError("per_env_cube_size with a placement_initializer: the cube's bottom offset would differ per environment")
        self.per_env_cube_size = per_env_cube_size
        self._cube_ov = None
        self._new_cube_size = None  # drawn by _sample_reset_state, written by _randomize_model
        self._cube_drawn = False
        super().__init__(*args, **kwargs)

    def _load_model(self, xml):
        return load_task_model("Lift", self.robot_name, xml)

    def _setup_references(self):
        super()._setup_references()
        m = self.model
        self.cube_body_id = m.names["body"].index("cube_main")
        self.cube_joint = m.names["joint"].index("cube_joint0")
        self.cube_qadr = int(m.jnt_qposadr[self.cube_joint])
        self.cube_geoms = [i for i, n in enumerate(m.names["geom"]) if n and n.startswith("cube_g")]
        self.cube_half_height = float(m.geom_size[self.cube_geoms[0], 2])

    def _setup_observables(self, ob):
        super()._setup_observables(ob)
        if self.use_object_obs:  # lift.py:356-399
            b, s = self.cube_body_id, self.eef_site_id
            ob.add("cube_pos", "object", [(OB_BODY_POS, b, k) for k in range(3)])
            ob.add("cube_quat", "object", [(OB_BODY_QUAT_XYZW, b, k) for k in range(4)])
            ob.add("gripper_to_cube_pos", "object", [(OB_BODY_MINUS_SITE, (b << 8) | s, k) for k in range(3)])

    def _setup_task(self):
        left, right = self._fingerpad_geoms()
        self.sim.task_config(self.cube_body_id, self.eef_site_id, left, right, self.cube_geoms)
        if self.per_env_cube_size:
            m, b = self.model, self.cube_body_id
            g = m.names["geom"].index("cube_g0")  # the colliding box; cube_g0_vis does not collide
            self._cube_ov = (self.sim.model_override("geom_size", g), self.sim.model_override("body_mass", b),
                             self.sim.model_override("body_inertia", b))
            # box moments are about the geom's axes; the engine wants them about the body's principal (inertial) axes, which
            # body_iquat rotates away from the geom's: moment k of the inertial frame = sum_j (R_i^T R_g)[k, j]^2 * moment j of the geom
            Ri, Rg = quat2mat(m.body_iquat[b]), quat2mat(m.geom_quat[g])
            self._cube_axis_map = (Ri.T @ Rg) ** 2

    def _placement_objects(self):
        """the cube as the reference's BoxObject: horizontal radius |half size[:2]|, bottom / top offsets -/+ half size z"""
        h = self.model.geom_size[self.model.names["geom"].index("cube_g0")]
        return {"cube": dict(radius=float(np.linalg.norm(h[:2])), bottom=-float(h[2]), top=float(h[2]), qpos_adr=self.cube_qadr, body=-1)}

    def _sample_reset_state(self, n):
        """robot: init_qpos + N(0, 0.02^2) (robots/robot.py:247-259); cube: x,y ~ U[-0.03,0.03], yaw ~ U[0,2pi),
        z = table + 0.01 + half height (lift.py:311-336, placement_samplers.py:221-309), or the placement_initializer's rules"""
        import torch

        q = self._robot_reset_qpos(n)
        if self.placement_initializer is not None:
            self._place_objects(q)
            return q
        u = torch.rand((n, 3), generator=self.rng, device=self.device, dtype=torch.float64)
        a = self.cube_qadr
        q[:, a] = self.table_offset[0] + (u[:, 0] * 2 - 1) * 0.03
        q[:, a + 1] = self.table_offset[1] + (u[:, 1] * 2 - 1) * 0.03
        half_height = self.cube_half_height
        if self._cube_ov is not None:
            # a new cube per environment when the model is rebuilt: at construction, and at every reset with hard_reset=True
            # (written to the masked environments by _randomize_model, which base.reset calls next)
            if not self._cube_drawn or self.hard_reset:
                lo, hi = self.cube_size_range
                self._new_cube_size = lo + (hi - lo) * torch.rand((n, 3), generator=self.rng, device=self.device, dtype=torch.float64)
                self._cube_drawn = True
                half_height = self._new_cube_size[:, 2]
            else:
                half_height = self._cube_ov[0][:, 2].to(device=self.device, dtype=torch.float64)
        q[:, a + 2] = self.table_offset[2] + 0.01 + half_height
        yaw = u[:, 2] * 2 * math.pi
        q[:, a + 3] = torch.cos(yaw / 2)
        q[:, a + 4] = 0
        q[:, a + 5] = 0
        q[:, a + 6] = torch.sin(yaw / 2)
        return q

    def _randomize_model(self, mask):
        """per-environment cube of the environments being reset (per_env_cube_size): size, mass 1000 * 8 * prod(size), box moments"""
        import torch

        if self._cube_ov is None or self._new_cube_size is None:
            return
        s, self._new_cube_size = self._new_cube_size, None
        mass = 8000.0 * s.prod(dim=1)
        box = torch.stack([s[:, 1] ** 2 + s[:, 2] ** 2, s[:, 0] ** 2 + s[:, 2] ** 2, s[:, 0] ** 2 + s[:, 1] ** 2], 1) * (mass / 3)[:, None]
        inertia = box @ self._dev_const("cube_axis_map", self._cube_axis_map).T
        for dst, src in zip(self._cube_ov, (s, mass, inertia)):
            src = src.to(device=dst.device, dtype=dst.dtype)
            if mask is None:
                dst.copy_(src)
            else:
                sel = mask.to(dst.device)
                dst.copy_(torch.where(sel[:, None] if src.ndim == 2 else sel, src, dst))

    def _check_success(self):
        """cube higher than the table top + 0.04 (lift.py:433-444); uses the pose of the last step1 like the reference"""
        return self.sim.task_out[:, 0] > self.table_offset[2] + 0.04

    def reward(self, action=None):
        """lift.py:224-273: 2.25 if lifted, else (shaping) reaching 1 - tanh(10 d) + 0.25 grasp; scaled by scale/2.25"""
        import torch

        t = self.sim.task_out
        success = self._check_success()
        r = torch.where(success, torch.full_like(t[:, 0], 2.25), torch.zeros_like(t[:, 0]))
        if self.reward_shaping:
            shaped = 1 - torch.tanh(10.0 * t[:, 1]) + 0.25 * t[:, 2]
            r = torch.where(success, r, shaped)
        if self.reward_scale is not None:
            r = r * (self.reward_scale / 2.25)
        return r
