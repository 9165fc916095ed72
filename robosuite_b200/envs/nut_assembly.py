"""NutAssembly tasks (robosuite/environments/manipulation/nut_assembly.py) on the batched engine."""
import math

import numpy as np

from .base import (OB_BODY_POS, OB_BODY_QUAT_XYZW, OB_SITE_POS, BatchedMujocoEnv, load_task_model, register_env)
from .single_object import SingleObjectMixin, parse_mode, reject_fixed

# models/assets/objects/{square,round}-nut.xml: bottom_site z, top_site z, horizontal_radius_site (x, y).  top_site (0, 0, 0.05) is
# recalled from robosuite v1.5 (no reference checkout was at hand); only a placement_initializer's overlap rule reads it
NUT_META = {"SquareNut": dict(bottom=-0.05, top=0.05, hradius=math.hypot(0.11, 0.06)),
            "RoundNut": dict(bottom=-0.05, top=0.05, hradius=math.hypot(0.11, 0.05))}


class _BatchedNutAssembly(SingleObjectMixin, BatchedMujocoEnv):
    """Both nuts are in the model (as in the reference).  single_object_mode 2 (NutAssemblySquare / NutAssemblyRound, or
    nut_type="square" / "round"): the unused nut is moved out of the scene at reset (environments/base.py:591-602 clear_objects ->
    (10, 10, 10)), where it drops onto the floor plane and rests.  single_object_mode 1 (NutAssemblySingle): one nut per environment,
    drawn at every reset (envs/single_object.py)."""

    table_offset = (0.0, 0.0, 0.82)  # nut_assembly.py:166
    maxcon, maxefc = 96, 288
    nut_names = ("SquareNut", "RoundNut")
    nut_to_id = {"square": 0, "round": 1}
    nut_id = 0
    _task_state = ("objects_on_pegs",)  # carried by get_env_state / set_env_state (mode 1's selection: by the engine's snapshot)

    def __init__(self, *args, single_object_mode=0, nut_type=None, **kwargs):
        self.single_object_mode, self._fixed_object = parse_mode(single_object_mode, nut_type, self.nut_to_id, "nut_type")
        if self._fixed_object is not None:
            self.nut_id = self._fixed_object
        self._object_names = self.nut_names
        super().__init__(*args, **kwargs)

    def _load_model(self, xml):
        return load_task_model("NutAssemblyRound", self.robot_name, xml)  # same composed model for all variants

    def _setup_references(self):
        super()._setup_references()
        m = self.model
        bn, jn, gn, sn = m.names["body"], m.names["joint"], m.names["geom"], m.names["site"]
        self.table_body_id, self.peg1_body_id, self.peg2_body_id = bn.index("table"), bn.index("peg1"), bn.index("peg2")
        self.obj_body_id = {n: bn.index(n + "_main") for n in self.nut_names}
        self.obj_qadr = {n: int(m.jnt_qposadr[jn.index(n + "_joint0")]) for n in self.nut_names}
        self.obj_geom_id = {n: [i for i, g in enumerate(gn) if g and g.startswith(n + "_g") and m.geom_contype[i]] for n in self.nut_names}
        self.object_site_ids = [sn.index(n + "_handle_site") for n in self.nut_names]
        self.active = [i for i in range(2) if self.single_object_mode != 2 or i == self.nut_id]
        self.objects_on_pegs = None
        self._setup_selection()

    def _setup_observables(self, ob):
        super()._setup_observables(ob)
        if self.use_object_obs and self.single_object_mode == 1:
            self._add_selected_object_obs(ob, "nut", "nut_id")
        elif self.use_object_obs:  # nut_assembly.py:478-580; inactive nuts' sensors are disabled, world_pose_in_gripper is inactive
            for i in self.active:
                n = self.nut_names[i]
                b = self.obj_body_id[n]
                ob.add_rel_pose(n, self.eef_site_id, self.eef_body_id, "object")
                ob.add(n + "_pos", "object", [(OB_BODY_POS, b, k) for k in range(3)])
                ob.add(n + "_quat", "object", [(OB_BODY_QUAT_XYZW, b, k) for k in range(4)])

    def _setup_task(self):
        left, right = self._fingerpad_geoms()
        n0 = self.nut_names[self.active[0]]
        self.sim.task_config(self.obj_body_id[n0], self.eef_site_id, left, right, self.obj_geom_id[n0])
        self.sim.task_objects([self.obj_geom_id[n] for n in self.nut_names])
        rows = [(OB_SITE_POS, self.eef_site_id, k) for k in range(3)]
        for i, n in enumerate(self.nut_names):
            rows += [(OB_BODY_POS, self.obj_body_id[n], k) for k in range(3)]
            rows += [(OB_SITE_POS, self.object_site_ids[i], k) for k in range(3)]
        self.sim.task_table(rows)  # eef(3), then per nut: body pos(3), handle site pos(3)
        self.peg_xy = [np.asarray(self.model.body_pos[b][:2], dtype=np.float64) for b in (self.peg1_body_id, self.peg2_body_id)]
        self.table_z = float(self.model.body_pos[self.table_body_id][2])

    def _placement_objects(self):
        """both nuts (also in the single-object variants, which park the unused one afterwards), in nut_assembly.py's order"""
        return {n: dict(radius=NUT_META[n]["hradius"], bottom=NUT_META[n]["bottom"], top=NUT_META[n]["top"], qpos_adr=self.obj_qadr[n],
                        body=-1) for n in self.nut_names}

    def _sample_reset_state(self, n):
        """nuts: x ~ U[-0.115, -0.11], y ~ U[0.11, 0.225] (square) / U[-0.225, -0.11] (round), yaw ~ U[0, 2pi),
        z = table + 0.02 - bottom_offset (nut_assembly.py:405-431, placement_samplers.py:255-309)"""
        import torch

        q = self._robot_reset_qpos(n)
        dev = self.device
        if self.placement_initializer is not None:
            self._place_objects(q)
            self._park_objects(q)
            return q
        for i, (name, yr) in enumerate(zip(self.nut_names, ((0.11, 0.225), (-0.225, -0.11)))):
            u = torch.rand((n, 3), generator=self.rng, device=dev, dtype=torch.float64)
            x = self.table_offset[0] + (-0.115 + u[:, 0] * 0.005)
            y = self.table_offset[1] + (yr[0] + u[:, 1] * (yr[1] - yr[0]))
            z = torch.full((n,), self.table_offset[2] + 0.02 - NUT_META[name]["bottom"], device=dev, dtype=torch.float64)
            self._place_free_body(q, self.obj_qadr[name], x, y, z, u[:, 2] * 2 * math.pi)
        self._park_objects(q)  # clear_objects
        return q

    def reset(self, mask=None, host_mask=None):
        import torch

        if self.objects_on_pegs is None:
            self.objects_on_pegs = torch.zeros((self.num_envs, 2), dtype=torch.bool, device=self.device)
        if mask is None:
            self.objects_on_pegs[:] = False
        else:
            self.objects_on_pegs.masked_fill_(mask.to(device=self.device, dtype=torch.bool)[:, None], False)
        return super().reset(mask, host_mask)

    # ---- reward machinery (nut_assembly.py:247-400, 614-640)
    def _task_views(self):
        t = self.sim.task_vec
        eef = t[:, 0:3]
        pos = [t[:, 3 + 6 * i:6 + 6 * i] for i in range(2)]
        handle = [t[:, 6 + 6 * i:9 + 6 * i] for i in range(2)]
        return eef, pos, handle

    def _update_on_pegs(self):
        import torch

        eef, pos, _ = self._task_views()
        for i in range(2):
            p = pos[i]
            peg = self.peg_xy[i]
            on = (torch.abs(p[:, 0] - peg[0]) < 0.03) & (torch.abs(p[:, 1] - peg[1]) < 0.03) & (p[:, 2] < self.table_offset[2] + 0.05)
            r_reach = 1 - torch.tanh(10.0 * torch.linalg.norm(eef - p, dim=1))
            self.objects_on_pegs[:, i] = on & (r_reach < 0.6)

    def _check_success(self):
        self._update_on_pegs()
        n = self.objects_on_pegs.sum(dim=1)
        return n > 0 if self.single_object_mode > 0 else n == 2

    def staged_rewards(self):
        """(r_reach, r_grasp, r_lift, r_hover); the reference iterates over ALL nuts not yet on their pegs (also the one
        parked at (10, 10, 10) in the single-nut variants)"""
        import torch

        reach_mult, grasp_mult, lift_mult, hover_mult = 0.1, 0.35, 0.5, 0.7
        eef, pos, handle = self._task_views()
        act = ~self.objects_on_pegs                                   # [N, 2]
        any_act = act.any(dim=1)
        big = torch.full_like(eef[:, 0], 1e9)
        dist = torch.stack([torch.where(act[:, i], torch.linalg.norm(handle[i] - eef, dim=1), big) for i in range(2)], dim=1)
        r_reach = torch.where(any_act, (1 - torch.tanh(10.0 * dist.min(dim=1).values)) * reach_mult, torch.zeros_like(big))
        bits = self.sim.task_out[:, 5].to(torch.int32)
        grasp = torch.zeros_like(any_act)
        for i in range(2):
            grasp |= act[:, i] & ((bits >> i) & 1).bool()
        r_grasp = grasp.to(eef.dtype) * grasp_mult
        z_target = self.table_z + 0.2
        zd = torch.stack([torch.where(act[:, i], torch.clamp(z_target - pos[i][:, 2], min=0.0), big) for i in range(2)], dim=1)
        r_lift = torch.where(any_act & grasp, grasp_mult + (1 - torch.tanh(15.0 * zd.min(dim=1).values)) * (lift_mult - grasp_mult),
                             torch.zeros_like(big))
        hov = []
        for i in range(2):
            peg = torch.as_tensor(self.peg_xy[i], device=self.device, dtype=eef.dtype)
            d = torch.linalg.norm(peg - pos[i][:, :2], dim=1)
            hov.append(torch.where(act[:, i], r_lift + (1 - torch.tanh(10.0 * d)) * (hover_mult - lift_mult), -big))
        r_hover = torch.where(any_act, torch.stack(hov, dim=1).max(dim=1).values, torch.zeros_like(big))
        return r_reach, r_grasp, r_lift, r_hover

    def reward(self, action=None):
        import torch

        self._check_success()
        r = self.objects_on_pegs.sum(dim=1).to(self.dtype)
        if self.reward_shaping:
            r = r + torch.stack(self.staged_rewards(), dim=1).max(dim=1).values.to(self.dtype)
        if self.reward_scale is not None:
            r = r * self.reward_scale
            if self.single_object_mode == 0:
                r = r / 2.0
        return r


@register_env
class BatchedNutAssembly(_BatchedNutAssembly):
    single_object_mode = 0


class _FixedNutAssembly(_BatchedNutAssembly):
    _mode = _type = None

    def __init__(self, *args, **kwargs):
        reject_fixed(kwargs, "single_object_mode", "nut_type")
        super().__init__(*args, single_object_mode=self._mode, nut_type=self._type, **kwargs)


@register_env
class BatchedNutAssemblySquare(_FixedNutAssembly):
    _mode, _type = 2, "square"


@register_env
class BatchedNutAssemblyRound(_FixedNutAssembly):
    _mode, _type = 2, "round"


@register_env
class BatchedNutAssemblySingle(_FixedNutAssembly):
    """NutAssembly with single_object_mode 1: one nut per environment, drawn at every reset"""
    _mode = 1
