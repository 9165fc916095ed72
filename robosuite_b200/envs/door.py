"""Door task (robosuite/environments/manipulation/door.py) on the batched engine."""
import math

import numpy as np

from .base import (OB_BODY_MINUS_SITE, OB_BODY_POS, OB_QPOS, OB_SITE_MINUS_SITE, OB_SITE_POS, BatchedMujocoEnv,
                   load_task_model, register_env)


@register_env
class BatchedDoor(BatchedMujocoEnv):
    """suite.make("Door", robots="Panda", num_envs=N): hinged door with a spring-loaded latch (use_latch=True, the
    reference default).  The reference draws the door pose per reset and writes it into model.body_pos/body_quat
    (door.py:303-318, 417-427); here the pose is per-environment DATA (`BatchedSim.body_pose_override`), drawn per environment and
    reset from the same ranges.  `door_placement=(x, y, yaw)` (or an explicit `model=`) pins one placement for every environment."""

    table_offset = (-0.2, -0.35, 0.8)  # door.py:177
    maxcon, maxefc = 48, 160
    tier_small = (8, 32)  # small tail tier: see BatchedMujocoEnv.tier_small

    # door.xml's bottom_site z (door.py:32 below), and its top_site z and horizontal_radius_site x, recalled from robosuite v1.5 (no
    # reference checkout was at hand); only a placement_initializer reads them
    DOOR_META = dict(radius=0.3, bottom=-0.3, top=0.3)

    def __init__(self, *args, door_placement=None, **kwargs):
        if kwargs.get("table_full_size") is not None or kwargs.get("table_friction") is not None:
            raise NotImplementedError("Door: table_full_size / table_friction: the reference's Door has a fixed (0.8, 0.3, 0.05) table "
                                      "and takes no table arguments")
        # (x, y, yaw) relative to table_offset; sampler ranges x [0.07, 0.09], y [-0.01, 0.01], yaw [-pi/2 - 0.25, -pi/2]
        if door_placement is not None and kwargs.get("placement_initializer") is not None:
            raise ValueError("door_placement pins the door; a placement_initializer samples it: give one of them")
        self._fixed_door = kwargs.get("placement_initializer") is None and (door_placement is not None or kwargs.get("model") is not None)
        self.door_placement = door_placement if door_placement is not None else (0.08, 0.0, -math.pi / 2 - 0.125)
        self._door_ov = None
        super().__init__(*args, **kwargs)

    def _load_model(self, xml):
        m = load_task_model("Door", self.robot_name, xml)
        b = m.names["body"].index("Door_main")
        x, y, yaw = self.door_placement
        # z: reference_pos z - bottom_offset z (door.xml bottom_site at -0.3), placement_samplers.py:277-279
        m.body_pos[b] = [self.table_offset[0] + x, self.table_offset[1] + y, self.table_offset[2] + 0.3]
        m.body_quat[b] = [math.cos(yaw / 2), 0.0, 0.0, math.sin(yaw / 2)]
        return m

    def _setup_references(self):
        super()._setup_references()
        m = self.model
        bn, jn = m.names["body"], m.names["joint"]
        self.door_body_id = bn.index("Door_door")
        self.frame_body_id = bn.index("Door_frame")
        self.latch_body_id = bn.index("Door_latch")
        self.door_handle_site_id = m.names["site"].index("Door_handle")
        self.hinge_qpos_addr = int(m.jnt_qposadr[jn.index("Door_hinge")])
        self.use_latch = "Door_latch_joint" in jn
        if self.use_latch:
            self.handle_qpos_addr = int(m.jnt_qposadr[jn.index("Door_latch_joint")])

    def _setup_observables(self, ob):
        super()._setup_observables(ob)
        if self.use_object_obs:  # door.py:345-398, in the reference's order
            d, h, s = self.door_body_id, self.door_handle_site_id, self.eef_site_id
            ob.add("door_pos", "object", [(OB_BODY_POS, d, k) for k in range(3)])
            ob.add("handle_pos", "object", [(OB_SITE_POS, h, k) for k in range(3)])
            ob.add("hinge_qpos", "object", [(OB_QPOS, self.hinge_qpos_addr, 0)])
            ob.add("door_to_eef_pos", "object", [(OB_BODY_MINUS_SITE, (d << 8) | s, k) for k in range(3)])
            ob.add("handle_to_eef_pos", "object", [(OB_SITE_MINUS_SITE, (h << 8) | s, k) for k in range(3)])
            if self.use_latch:
                ob.add("handle_qpos", "object", [(OB_QPOS, self.handle_qpos_addr, 0)])

    def _setup_task(self):
        left, right = self._fingerpad_geoms()
        self.sim.task_config(self.door_body_id, self.eef_site_id, left, right, [])
        h, s = self.door_handle_site_id, self.eef_site_id
        self.sim.task_table([(OB_SITE_MINUS_SITE, (h << 8) | s, k) for k in range(3)])  # _gripper_to_handle after the step
        if not self._fixed_door:
            bn = self.model.names["body"]
            main, frame = bn.index("Door_main"), bn.index("Door_frame")
            self._door_ov = (self.sim.body_pose_override(main), self.sim.body_pose_override(frame))
            self._frame_local = (np.asarray(self.model.body_pos[frame], dtype=np.float64), np.asarray(self.model.body_quat[frame], dtype=np.float64))

    @property
    def door_pose(self):
        """(pos [N, 3], quat [N, 4] wxyz) of the door's root body per environment, or None with a pinned placement"""
        return None if self._door_ov is None else self._door_ov[0]

    def _placement_objects(self):
        """the door's root body, placed through its world-pose override (and Door_frame's, welded to it)"""
        return {"Door": dict(self.DOOR_META, qpos_adr=-1, body=self.model.names["body"].index("Door_main"))}

    def _randomize_model(self, mask):
        """UniformRandomSampler of door.py:303-318: x in [0.07, 0.09], y in [-0.01, 0.01], yaw in [-pi/2 - 0.25, -pi/2] about z,
        relative to table_offset; z = table height + 0.3 (the door's bottom offset).  A placement_initializer's placement was
        written by _sample_reset_state instead."""
        import torch

        if self._door_ov is None or self.placement_initializer is not None:
            return
        n, dev = self.num_envs, self.device
        u = torch.rand((n, 3), generator=self.rng, device=dev, dtype=torch.float64)
        x = self.table_offset[0] + 0.07 + 0.02 * u[:, 0]
        y = self.table_offset[1] - 0.01 + 0.02 * u[:, 1]
        yaw = (-math.pi / 2 - 0.25) + 0.25 * u[:, 2]
        z = torch.full_like(x, self.table_offset[2] + 0.3)
        c, s_ = torch.cos(yaw / 2), torch.sin(yaw / 2)
        zero = torch.zeros_like(x)
        pos_m = torch.stack([x, y, z], 1)
        quat_m = torch.stack([c, zero, zero, s_], 1)
        lp, lq = self._dev_const("door_frame_lp", self._frame_local[0]), self._dev_const("door_frame_lq", self._frame_local[1])
        cy, sy = torch.cos(yaw), torch.sin(yaw)
        pos_f = pos_m + torch.stack([cy * lp[0] - sy * lp[1], sy * lp[0] + cy * lp[1], zero + lp[2]], 1)
        # (c, 0, 0, s) * (w, x, y, z)
        quat_f = torch.stack([c * lq[0] - s_ * lq[3], c * lq[1] - s_ * lq[2], c * lq[2] + s_ * lq[1], c * lq[3] + s_ * lq[0]], 1)
        (pm, qm), (pf, qf) = self._door_ov
        for dst, src in ((pm, pos_m), (qm, quat_m), (pf, pos_f), (qf, quat_f)):
            src = src.to(device=dst.device, dtype=dst.dtype)
            if mask is None:
                dst.copy_(src)
            else:
                dst.copy_(torch.where(mask.to(dst.device)[:, None], src, dst))

    def _sample_reset_state(self, n):
        q = self._robot_reset_qpos(n)  # door closed, latch at rest (qpos0)
        if self.placement_initializer is not None:
            self._place_objects(q)  # the door's pose overrides
        return q

    def _check_success(self):
        """hinge opened beyond 0.3 rad (door.py:429-437); qpos after the step, as the reference reads it"""
        return self.sim.qpos[:, self.hinge_qpos_addr] > 0.3

    def reward(self, action=None):
        """door.py:219-266: 1 if opened; shaping: 0.25 (1 - tanh(10 |handle - eef|)) + latch rotation term"""
        import torch

        success = self._check_success()
        r = success.to(self.dtype)
        if self.reward_shaping:
            shaped = 0.25 * (1 - torch.tanh(10.0 * torch.linalg.norm(self.sim.task_vec, dim=1)))
            if self.use_latch:
                hq = self.sim.qpos[:, self.handle_qpos_addr]
                shaped = shaped + torch.clamp(0.25 * torch.abs(hq / (0.5 * np.pi)), -0.25, 0.25)
            r = torch.where(success, r, shaped.to(self.dtype))
        if self.reward_scale is not None:
            r = r * (self.reward_scale / 1.0)
        return r
