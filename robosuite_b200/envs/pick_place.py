"""PickPlace task (robosuite/environments/manipulation/pick_place.py) on the batched engine."""
import math

import numpy as np

from .base import OB_BODY_POS, OB_BODY_QUAT_XYZW, OB_SITE_POS, BatchedMujocoEnv, load_task_model, register_env
from .single_object import SingleObjectMixin, parse_mode, reject_fixed

# models/assets/objects/{milk,bread,cereal,can}.xml: bottom_site z, top_site z, horizontal_radius_site (x, y)
OBJ_META = {
    "Milk": dict(bottom=-0.085, top=0.075, hradius=math.hypot(0.025, 0.025)),
    "Bread": dict(bottom=-0.045, top=0.03, hradius=math.hypot(0.03, 0.03)),
    "Cereal": dict(bottom=-0.10, top=0.03, hradius=math.hypot(0.04, 0.03)),
    "Can": dict(bottom=-0.06, top=0.04, hradius=math.hypot(0.025, 0.025)),
}


@register_env
class BatchedPickPlace(SingleObjectMixin, BatchedMujocoEnv):
    """suite.make("PickPlace", robots="Panda", num_envs=N, single_object_mode=0, object_type=None): four objects in bin 1, one
    target quadrant each in bin 2.  single_object_mode 1 (one object drawn per environment at every reset) and 2 (the object
    `object_type`: "milk", "bread", "cereal" or "can"): see envs/single_object.py.  The visual target objects have no physics and are
    not modelled."""

    obj_names = ("Milk", "Bread", "Cereal", "Can")
    object_to_id = {"milk": 0, "bread": 1, "cereal": 2, "can": 3}
    maxcon, maxefc = 64, 224
    tier_small = (12, 56)  # small tail tier: see BatchedMujocoEnv.tier_small
    _task_state = ("objects_in_bins",)  # carried by get_env_state / set_env_state (mode 1's selection: by the engine's snapshot)

    bin1_pos = np.array([0.1, -0.25, 0.8])   # pick_place.py:186-187 (pinned: the packaged model's bin1 / bin2 bodies)
    bin2_pos = np.array([0.1, 0.28, 0.8])
    bin_size = np.array([0.39, 0.49, 0.82])  # BinsArena table_full_size (pick_place.py:184)
    table_full_size_default = (0.39, 0.49, 0.82)
    table_friction_default = (1.0, 5e-3, 1e-4)
    _table_args_refused = "the bins arena's wall geometry for another table is not known here"

    def __init__(self, *args, single_object_mode=0, object_type=None, bin1_pos=None, bin2_pos=None, z_offset=0.0, z_rotation=None,
                 **kwargs):
        """bin1_pos / bin2_pos: world positions of the two bins (bin 1 holds the objects at reset, bin 2 the targets and the success
        regions); z_offset: added to every object's placement height; z_rotation: the placement yaw, None = U[0, 2 pi), a number = that
        angle, a (lo, hi) pair = U[lo, hi) (the reference's UniformRandomSampler `rotation`, recalled from robosuite v1.5).  The bins
        are moved in the model, for every environment; the robot base stays where the bins arena puts it."""
        self.bin1_pos = self._position("bin1_pos", bin1_pos, type(self).bin1_pos)
        self.bin2_pos = self._position("bin2_pos", bin2_pos, type(self).bin2_pos)
        if not (isinstance(z_offset, (int, float, np.floating, np.integer)) and math.isfinite(float(z_offset))):
            raise ValueError("z_offset must be a finite number, got {!r}".format(z_offset))
        self.z_offset = float(z_offset)
        self.z_rotation = self._rotation(z_rotation)
        self.single_object_mode, self._fixed_object = parse_mode(single_object_mode, object_type, self.object_to_id, "object_type")
        self._object_names = self.obj_names
        if self.single_object_mode:
            # the parked objects resting on the floor add contacts: 13 on average at 4096 environments under random actions, 16 - 17 at
            # the 99.9th percentile (tools/probe_instr.py on an H100), where (12, 56) left 99.9 % of the environment-substeps to the large tier
            self.tier_small = (18, 80)
        super().__init__(*args, **kwargs)

    @staticmethod
    def _position(name, v, default):
        if v is None:
            return default
        a = np.array(v, dtype=np.float64)
        if a.shape != (3,) or not np.all(np.isfinite(a)):
            raise ValueError("{} must be 3 finite numbers, got {!r}".format(name, v))
        return a

    @staticmethod
    def _rotation(r):
        """z_rotation as None or a (lo, hi) pair (a number: (a, a))"""
        if r is None:
            return None
        a = np.array(r, dtype=np.float64)
        if a.shape == ():
            a = np.array([a, a])
        if a.shape != (2,) or not np.all(np.isfinite(a)):
            raise ValueError("z_rotation must be None, a finite number or a (lo, hi) pair, got {!r}".format(r))
        return float(a.min()), float(a.max())

    def _load_model(self, xml):
        return load_task_model("PickPlace", self.robot_name, xml)

    def _arena_model(self, model):
        """bin1 / bin2 bodies at bin1_pos / bin2_pos (world-welded, children of the world); the defaults leave the model untouched"""
        import copy

        moved = [(n, p) for n, p, d in (("bin1", self.bin1_pos, type(self).bin1_pos), ("bin2", self.bin2_pos, type(self).bin2_pos))
                 if not np.array_equal(p, d)]
        if not moved:
            return model
        m = copy.copy(model)
        m.body_pos = np.array(model.body_pos, dtype=np.float64)
        for n, p in moved:
            m.body_pos[m.names["body"].index(n)] = p
        return m

    def _setup_references(self):
        super()._setup_references()
        m = self.model
        bn, jn, gn = m.names["body"], m.names["joint"], m.names["geom"]
        self.obj_body_id = {n: bn.index(n + "_main") for n in self.obj_names}
        self.obj_qadr = {n: int(m.jnt_qposadr[jn.index(n + "_joint0")]) for n in self.obj_names}
        self.obj_geom_id = {n: [i for i, g in enumerate(gn) if g and g.startswith(n + "_g") and m.geom_contype[i]] for n in self.obj_names}
        # target_bin_placements (pick_place.py:570-583)
        tb = np.zeros((4, 3))
        for i in range(4):
            x, y = self.bin2_pos[0], self.bin2_pos[1]
            if i in (0, 2):
                x -= self.bin_size[0] / 2.0
            if i < 2:
                y -= self.bin_size[1] / 2.0
            tb[i] = [x + self.bin_size[0] / 4.0, y + self.bin_size[1] / 4.0, self.bin2_pos[2]]
        self.target_bin_placements = tb
        self.objects_in_bins = None
        self._setup_selection()

    def _setup_observables(self, ob):
        super()._setup_observables(ob)
        if self.use_object_obs and self.single_object_mode == 1:
            self._add_selected_object_obs(ob, "obj", "obj_id")
        elif self.use_object_obs:  # pick_place.py:585-685; mode 2: the fixed object's observables only
            for i, n in enumerate(self.obj_names):
                if self.single_object_mode == 2 and i != self._fixed_object:
                    continue
                b = self.obj_body_id[n]
                ob.add_rel_pose(n, self.eef_site_id, self.eef_body_id, "object")
                ob.add(n + "_pos", "object", [(OB_BODY_POS, b, k) for k in range(3)])
                ob.add(n + "_quat", "object", [(OB_BODY_QUAT_XYZW, b, k) for k in range(4)])

    def _setup_task(self):
        left, right = self._fingerpad_geoms()
        n0 = self.obj_names[0]
        self.sim.task_config(self.obj_body_id[n0], self.eef_site_id, left, right, self.obj_geom_id[n0])
        self.sim.task_objects([self.obj_geom_id[n] for n in self.obj_names])
        rows = [(OB_SITE_POS, self.eef_site_id, k) for k in range(3)]
        for n in self.obj_names:
            rows += [(OB_BODY_POS, self.obj_body_id[n], k) for k in range(3)]
        self.sim.task_table(rows)  # eef(3), then body pos(3) per object

    def _sample_reset_state(self, n):
        """objects one after the other, uniformly in bin 1 with the footprint inside the bin and no overlap with the
        objects placed before (UniformRandomSampler: placement_samplers.py:255-309; pick_place.py:428-450)"""
        import torch

        q = self._robot_reset_qpos(n)
        dev = self.device
        hx, hy = self.bin_size[0] / 2 - 0.05, self.bin_size[1] / 2 - 0.05
        placed = []
        for name in self.obj_names:
            meta = OBJ_META[name]
            r = meta["hradius"]
            z = float((self.z_offset + self.bin1_pos[2]) - meta["bottom"])

            # R candidate positions per environment, the first one that clears every object placed before is taken: the distribution of the
            # reference's sequential rejection loop without a device->host round trip per attempt (no candidate fits: < 1e-12 per reset)
            R = 64
            u = torch.rand((R, n, 2), generator=self.rng, device=dev, dtype=torch.float64)
            cx = self.bin1_pos[0] + (-hx + r) + u[..., 0] * 2 * (hx - r)
            cy = self.bin1_pos[1] + (-hy + r) + u[..., 1] * 2 * (hy - r)
            ok = torch.ones((R, n), dtype=torch.bool, device=dev)
            for (px, py, pz, pmeta) in placed:
                if z - pz <= pmeta["top"] - meta["bottom"]:
                    ok &= (cx - px) ** 2 + (cy - py) ** 2 > (pmeta["hradius"] + r) ** 2
            ok[R - 1] = True
            first = torch.argmax(ok.to(torch.uint8), dim=0, keepdim=True)
            x, y = torch.gather(cx, 0, first)[0], torch.gather(cy, 0, first)[0]
            yaw = torch.rand((n,), generator=self.rng, device=dev, dtype=torch.float64)
            if self.z_rotation is None:
                yaw = yaw * 2 * math.pi
            else:
                lo, hi = self.z_rotation
                yaw = lo + yaw * (hi - lo) if hi > lo else torch.full_like(yaw, lo)
            self._place_free_body(q, self.obj_qadr[name], x, y, torch.full((n,), z, device=dev, dtype=torch.float64), yaw)
            placed.append((x, y, z, meta))
        self._park_objects(q)
        return q

    def reset(self, mask=None, host_mask=None):
        import torch

        if self.objects_in_bins is None:
            self.objects_in_bins = torch.zeros((self.num_envs, 4), dtype=torch.bool, device=self.device)
        if mask is None:
            self.objects_in_bins[:] = False
        else:
            self.objects_in_bins.masked_fill_(mask.to(device=self.device, dtype=torch.bool)[:, None], False)
        return super().reset(mask, host_mask)

    # ---- reward machinery (pick_place.py:275-425, 728-750)
    def _task_views(self):
        t = self.sim.task_vec
        return t[:, 0:3], [t[:, 3 + 3 * i:6 + 3 * i] for i in range(4)]

    def _bin_bounds(self, i):
        x, y = self.bin2_pos[0], self.bin2_pos[1]
        if i in (0, 2):
            x -= self.bin_size[0] / 2
        if i < 2:
            y -= self.bin_size[1] / 2
        return x, x + self.bin_size[0] / 2, y, y + self.bin_size[1] / 2

    def _update_in_bins(self):
        import torch

        eef, pos = self._task_views()
        for i in range(4):
            p = pos[i]
            xl, xh, yl, yh = self._bin_bounds(i)
            inside = (p[:, 0] > xl) & (p[:, 0] < xh) & (p[:, 1] > yl) & (p[:, 1] < yh) & (p[:, 2] > self.bin2_pos[2]) & (p[:, 2] < self.bin2_pos[2] + 0.1)
            r_reach = 1 - torch.tanh(10.0 * torch.linalg.norm(eef - p, dim=1))
            self.objects_in_bins[:, i] = inside & (r_reach < 0.6)

    def _check_success(self):
        self._update_in_bins()
        n = self.objects_in_bins.sum(dim=1)
        return n > 0 if self.single_object_mode > 0 else n == 4

    def staged_rewards(self):
        import torch

        reach_mult, grasp_mult, lift_mult, hover_mult = 0.1, 0.35, 0.5, 0.7
        eef, pos = self._task_views()
        act = ~self.objects_in_bins
        any_act = act.any(dim=1)
        zero = torch.zeros_like(eef[:, 0])
        big = torch.full_like(zero, 1e9)
        dist = torch.stack([torch.where(act[:, i], torch.linalg.norm(pos[i] - eef, dim=1), big) for i in range(4)], dim=1)
        r_reach = torch.where(any_act, (1 - torch.tanh(10.0 * dist.min(dim=1).values)) * reach_mult, zero)
        bits = self.sim.task_out[:, 5].to(torch.int32)
        grasp = torch.zeros_like(any_act)
        for i in range(4):
            grasp |= act[:, i] & ((bits >> i) & 1).bool()
        r_grasp = grasp.to(eef.dtype) * grasp_mult
        z_target = float(self.bin2_pos[2]) + 0.25
        zd = torch.stack([torch.where(act[:, i], torch.clamp(z_target - pos[i][:, 2], min=0.0), big) for i in range(4)], dim=1)
        r_lift = torch.where(any_act & grasp, grasp_mult + (1 - torch.tanh(15.0 * zd.min(dim=1).values)) * (lift_mult - grasp_mult), zero)
        hov = []
        for i in range(4):
            tx, ty = float(self.target_bin_placements[i, 0]), float(self.target_bin_placements[i, 1])
            above = (torch.abs(pos[i][:, 0] - tx) < self.bin_size[0] / 4.0) & (torch.abs(pos[i][:, 1] - ty) < self.bin_size[1] / 4.0)
            d = torch.sqrt((pos[i][:, 0] - tx) ** 2 + (pos[i][:, 1] - ty) ** 2)
            h = torch.where(above, lift_mult + (1 - torch.tanh(10.0 * d)) * (hover_mult - lift_mult),
                            r_lift + (1 - torch.tanh(10.0 * d)) * (hover_mult - lift_mult))
            hov.append(torch.where(act[:, i], h, -big))
        r_hover = torch.where(any_act, torch.stack(hov, dim=1).max(dim=1).values, zero)
        return r_reach, r_grasp, r_lift, r_hover

    def reward(self, action=None):
        import torch

        self._check_success()
        r = self.objects_in_bins.sum(dim=1).to(self.dtype)
        if self.reward_shaping:
            r = r + torch.stack(self.staged_rewards(), dim=1).max(dim=1).values.to(self.dtype)
        if self.reward_scale is not None:
            r = r * self.reward_scale / 4.0 if self.single_object_mode == 0 else r * self.reward_scale
        return r


class _FixedPickPlace(BatchedPickPlace):
    _mode = _type = None

    def __init__(self, *args, **kwargs):
        reject_fixed(kwargs, "single_object_mode", "object_type")
        super().__init__(*args, single_object_mode=self._mode, object_type=self._type, **kwargs)


@register_env
class BatchedPickPlaceSingle(_FixedPickPlace):
    """PickPlace with single_object_mode 1: one object per environment, drawn at every reset"""
    _mode = 1


@register_env
class BatchedPickPlaceMilk(_FixedPickPlace):
    _mode, _type = 2, "milk"


@register_env
class BatchedPickPlaceBread(_FixedPickPlace):
    _mode, _type = 2, "bread"


@register_env
class BatchedPickPlaceCereal(_FixedPickPlace):
    _mode, _type = 2, "cereal"


@register_env
class BatchedPickPlaceCan(_FixedPickPlace):
    """the "Can" task of the robomimic benchmarks"""
    _mode, _type = 2, "can"
