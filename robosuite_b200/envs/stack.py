"""Stack task (robosuite/environments/manipulation/stack.py) on the batched engine."""
import math

import numpy as np

from .base import (OB_BODY_MINUS_BODY, OB_BODY_MINUS_SITE, OB_BODY_POS, OB_BODY_QUAT_XYZW, BatchedMujocoEnv,
                   load_task_model, register_env)
from .lift import GRIPPER_INIT_QPOS, PANDA_INIT_QPOS, SAWYER_INIT_QPOS


@register_env
class BatchedStack(BatchedMujocoEnv):
    """suite.make("Stack", robots="Sawyer", num_envs=N): red cube A (2 cm) to be stacked on green cube B (2.5 cm)"""

    maxcon, maxefc = 48, 128
    tier_small = (12, 48)  # small tail tier: see BatchedMujocoEnv.tier_small (two cubes at rest: 8 contacts, 33-37 rows)

    table_offset = (0.0, 0.0, 0.8)  # stack.py:154

    def _load_model(self, xml):
        return load_task_model("Stack", self.robot_name, xml)

    def _setup_references(self):
        super()._setup_references()
        m = self.model
        bn, jn, gn = m.names["body"], m.names["joint"], m.names["geom"]
        self.cubeA_body_id, self.cubeB_body_id = bn.index("cubeA_main"), bn.index("cubeB_main")
        self.cubeA_qadr = int(m.jnt_qposadr[jn.index("cubeA_joint0")])
        self.cubeB_qadr = int(m.jnt_qposadr[jn.index("cubeB_joint0")])
        self.cubeA_geoms = [gn.index("cubeA_g0")]
        self.cubeB_geoms = [gn.index("cubeB_g0")]
        self.half = {"A": m.geom_size[self.cubeA_geoms[0]].copy(), "B": m.geom_size[self.cubeB_geoms[0]].copy()}

    def _setup_observables(self, ob):
        super()._setup_observables(ob)
        if self.use_object_obs:  # stack.py:423-470, in the reference's order
            A, B, s = self.cubeA_body_id, self.cubeB_body_id, self.eef_site_id
            ob.add("cubeA_pos", "object", [(OB_BODY_POS, A, k) for k in range(3)])
            ob.add("cubeA_quat", "object", [(OB_BODY_QUAT_XYZW, A, k) for k in range(4)])
            ob.add("cubeB_pos", "object", [(OB_BODY_POS, B, k) for k in range(3)])
            ob.add("cubeB_quat", "object", [(OB_BODY_QUAT_XYZW, B, k) for k in range(4)])
            ob.add("cubeA_to_cubeB", "object", [(OB_BODY_MINUS_BODY, (B << 8) | A, k) for k in range(3)])
            ob.add("gripper_to_cubeA", "object", [(OB_BODY_MINUS_SITE, (A << 8) | s, k) for k in range(3)])
            ob.add("gripper_to_cubeB", "object", [(OB_BODY_MINUS_SITE, (B << 8) | s, k) for k in range(3)])

    def _setup_task(self):
        left, right = self._fingerpad_geoms()
        self.sim.task_config(self.cubeA_body_id, self.eef_site_id, left, right, self.cubeA_geoms)
        self.sim.task_config2(self.cubeB_body_id, self.cubeB_geoms)

    def _placement_objects(self):
        """both cubes as the reference's BoxObject (horizontal radius |half size[:2]|, bottom / top offsets -/+ half size z), in
        stack.py's order"""
        return {"cube" + k: dict(radius=float(np.linalg.norm(self.half[k][:2])), bottom=-float(self.half[k][2]), top=float(self.half[k][2]),
                                 qpos_adr=getattr(self, "cube%s_qadr" % k), body=-1) for k in ("A", "B")}

    def _sample_reset_state(self, n):
        """robot init pose + noise; cubes: UniformRandomSampler x,y ~ U[-0.08,0.08], yaw ~ U[0,2pi), z = table + 0.01 +
        half height, cube B re-drawn while it overlaps cube A (placement_samplers.py:255-309, stack.py:357-388), or the
        placement_initializer's rules"""
        import torch

        dev = self.device
        q = self._robot_reset_qpos(n)
        if self.placement_initializer is not None:
            self._place_objects(q)
            return q

        def draw(*shape):
            u = torch.rand(shape + (3,), generator=self.rng, device=dev, dtype=torch.float64)
            return (u[..., 0] * 2 - 1) * 0.08, (u[..., 1] * 2 - 1) * 0.08, u[..., 2] * 2 * math.pi

        ax, ay, ayaw = draw(n)
        # cube B: the reference re-draws until the bounding circles are disjoint (placement_samplers.py:255-309; ~half of the draws collide).
        # Here R candidate placements are drawn per environment at once and the first valid one is taken - the same distribution as the
        # sequential rejection loop, with no device->host round trip per attempt (this runs inside step() for the auto-reset).  With R = 48
        # the probability that no candidate fits is < 1e-14 per reset; such an environment keeps its last candidate.
        R = 48
        cx, cy, cyaw = draw(R, n)
        rA = float(np.linalg.norm(self.half["A"][:2])); rB = float(np.linalg.norm(self.half["B"][:2]))
        ok = torch.sqrt((ax - cx) ** 2 + (ay - cy) ** 2) > rA + rB
        ok[R - 1] = True
        first = torch.argmax(ok.to(torch.uint8), dim=0, keepdim=True)  # index of the first valid candidate
        bx, by, byaw = (torch.gather(c, 0, first)[0] for c in (cx, cy, cyaw))
        for adr, x, y, yaw, hz in ((self.cubeA_qadr, ax, ay, ayaw, self.half["A"][2]), (self.cubeB_qadr, bx, by, byaw, self.half["B"][2])):
            q[:, adr] = self.table_offset[0] + x
            q[:, adr + 1] = self.table_offset[1] + y
            q[:, adr + 2] = self.table_offset[2] + 0.01 + float(hz)
            q[:, adr + 3] = torch.cos(yaw / 2)
            q[:, adr + 4] = 0
            q[:, adr + 5] = 0
            q[:, adr + 6] = torch.sin(yaw / 2)
        return q

    def staged_rewards(self):
        """(r_reach, r_lift, r_stack) of stack.py:266-312 from the kernel's task outputs"""
        import torch

        t = self.sim.task_out
        grasp = t[:, 2] > 0
        r_reach = (1 - torch.tanh(10.0 * t[:, 1])) * 0.25 + 0.25 * grasp
        lifted = t[:, 0] > self.table_offset[2] + 0.04
        r_lift = torch.where(lifted, 1.0 + 0.5 * (1 - torch.tanh(t[:, 3])), torch.zeros_like(t[:, 0]))
        r_stack = torch.where((~grasp) & (r_lift > 0) & (t[:, 4] > 0), torch.full_like(t[:, 0], 2.0), torch.zeros_like(t[:, 0]))
        return r_reach, r_lift, r_stack

    def _check_success(self):
        return self.staged_rewards()[2] > 0

    def reward(self, action=None):
        import torch

        r_reach, r_lift, r_stack = self.staged_rewards()
        if self.reward_shaping:
            r = torch.maximum(torch.maximum(r_reach, r_lift), r_stack)
        else:
            r = torch.where(r_stack > 0, torch.full_like(r_stack, 2.0), torch.zeros_like(r_stack))
        if self.reward_scale is not None:
            r = r * (self.reward_scale / 2.0)
        return r
