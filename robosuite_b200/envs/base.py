"""Batched environment API: the reference's MujocoEnv surface (`make`, `reset`, `step`, `_get_observations`,
`action_spec`, `reward`, `_check_success`) over N environments living on one GPU.

Behavioural spec, file:line in the reference:
  make / registry            robosuite/environments/base.py:23-56
  reset                      robosuite/environments/base.py:277-347 (+ robots/robot.py:234-300)
  step (25-substep loop)     robosuite/environments/base.py:467-521
  _get_observations          robosuite/environments/base.py:429-465
  action_spec                robosuite/environments/robot_env.py:271-285
The substep loop, controller, observation sampling and task outputs run inside ONE CUDA kernel per control step
(csrc/b2s_kernel.cuh); this module only assembles tensors.
"""
import os
from collections import OrderedDict

import numpy as np

from .. import controller_config as cc
from ..engine import BatchedSim, CtrlCfg
from ..mjcf.compiler import Model, compile_mjcf, load_model
from .contacts import ContactQueries

REGISTERED_ENVS = {}
_ASSETS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "assets", "models")

# observation scalar ops (must match enum OB_* in csrc/b2s_types.cuh)
OB_QPOS, OB_COS_QPOS, OB_SIN_QPOS, OB_QVEL, OB_QACC, OB_SITE_POS, OB_BODY_POS, OB_BODY_QUAT_XYZW, OB_SITE_QUAT_XYZW, \
    OB_BODY_MINUS_SITE, OB_SITE_MINUS_SITE, OB_BODY_QUAT_REL_SITE_XYZW, OB_ZERO, OB_BODY_MINUS_BODY, OB_REL_POS_LAG, \
    OB_REL_QUAT_LAG, OB_SEL_BODY_POS, OB_SEL_BODY_QUAT_XYZW, OB_SEL_INDEX = range(19)


def register_env(cls):
    REGISTERED_ENVS[cls.__name__.replace("Batched", "")] = cls
    return cls


def make(env_name, *args, **kwargs):
    """suite.make(env_name, robots=..., num_envs=N, **kw) (environments/base.py:23-42)"""
    if env_name not in REGISTERED_ENVS:
        raise Exception("Environment {} not found. Make sure it is a registered environment among: {}".format(
            env_name, ", ".join(REGISTERED_ENVS)))
    return REGISTERED_ENVS[env_name](*args, **kwargs)


def load_task_model(task, robot, xml=None):
    """Compiled model for task/robot: from a composed MJCF string (reference composer output) when given, else the
    packaged compiled fixture (mesh files do not travel to GPU boxes)."""
    if xml is not None:
        return compile_mjcf(xml)
    path = os.path.join(_ASSETS, f"{task}_{robot}.npz")
    if not os.path.exists(path):
        raise FileNotFoundError(f"no packaged model for {task}/{robot}; pass the composed MJCF via xml=")
    return load_model(path)


class ObsBuilder:
    """Collects (name, modality, op table rows) in the reference's observable order."""

    def __init__(self):
        self.items = []  # (name, modality, [(op,a,b),...])

    def add(self, name, modality, rows):
        self.items.append((name, modality, rows))

    def add_rel_pose(self, obj_key, eef_site, eef_body, modality, pf="robot0_"):
        """`{obj}_to_{pf}eef_pos` (3) and `{obj}_to_{pf}eef_quat` (4): pose of the object in the gripper frame, from the
        `{obj}_pos` / `{obj}_quat` values of the previous sample (manipulation_env.py:268-329).  The slots of those two
        observables are resolved in tables(), so they may be added afterwards, as the reference orders them."""
        b = (eef_site << 8) | (eef_body << 16)
        self.items.append((f"{obj_key}_to_{pf}eef_pos", modality, [("lagpos", obj_key, b | k) for k in range(3)]))
        self.items.append((f"{obj_key}_to_{pf}eef_quat", modality, [("lagquat", obj_key, b | k) for k in range(4)]))

    def tables(self):
        """rows ordered modality by modality (first-seen order), as _get_observations concatenates them"""
        mods = []
        for _, mod, _ in self.items:
            if mod not in mods:
                mods.append(mod)
        ops, slices, mod_slices = [], OrderedDict(), OrderedDict()
        for mod in mods:
            start = len(ops)
            for name, m2, rows in self.items:
                if m2 != mod:
                    continue
                slices[name] = (len(ops), len(ops) + len(rows))
                ops += rows
            mod_slices[mod + "-state"] = (start, len(ops))
        for i, row in enumerate(ops):
            if row[0] in ("lagpos", "lagquat"):
                ps, qs = slices[row[1] + "_pos"][0], slices[row[1] + "_quat"][0]
                ops[i] = (OB_REL_POS_LAG if row[0] == "lagpos" else OB_REL_QUAT_LAG, ps | (qs << 12), row[2])
        arr = np.array(ops, dtype=np.int32).reshape(-1, 3)
        return arr[:, 0], arr[:, 1], arr[:, 2], slices, mod_slices


# bits of sim.warn / info["sim_warn"] (robosuite_b200/csrc: b2s_kernel.cuh, b2s_collide.cuh, b2s_solver.cuh)
SIM_WARN_BITS = {1: "singular mass matrix", 2: "non-finite state in the integrator", 4: "contact capacity overflow (maxcon)",
                 8: "constraint-row capacity overflow (maxefc)", 16: "singular Newton Hessian",
                 32: "diverged state (non-finite / huge qpos, qvel or qacc): data reset to the model defaults, as mj_checkPos/Vel/Acc do",
                 64: "unit-queue watchdog fired: the control step is incomplete (mode 2 only; a library bug, please report)",
                 128: "invalid model override (non-finite or non-positive size, friction, mass or moment, moments violating the "
                      "triangle inequality, non-finite or negative damping, armature or friction loss, or a non-finite solref / "
                      "solimp component)",
                 256: "restore source row out of range (b2s_restore): the environment was left untouched",
                 512: "object selection out of range (obj_sel, b2s_obs_objects): the selected-object observation rows were written as 0",
                 1024: "no valid placement (placement_initializer, b2s_place_objects): an object kept its last of 5000 tries, where the "
                       "reference raises RandomizationError"}


# The reference's TableArena and robot base placement, recalled from robosuite v1.5 (models/arenas/table_arena.py,
# models/robots/manipulators/{panda,sawyer}_robot.py base_xpos_offset["table"]); no reference checkout was available.  Pinned by the
# packaged models, which the reference composer produced with the default arguments (tests/test_cpu_arena.py checks each):
#   table body pos    = table_offset - (0, 0, table_full_size[2] / 2)        (0.775 in Lift / Stack / Door, 0.795 in NutAssembly)
#   table_collision   = box, half sizes table_full_size / 2, friction table_friction   (0.4 0.4 0.025; 1 0.005 1e-4)
#   robot0_base pos x = -0.16 - table_full_size[0] / 2, y and z unchanged     (-0.56 everywhere, Door's 0.8-long table included)
# Recalled only: that the top of the table stays at table_offset[2] for every thickness, and that the legs are visual (they are
# not modelled here: no geom of theirs collides).
TABLE_GEOM, TABLE_BODY, ROBOT_ROOT = "table_collision", "table", "robot0_base"


def _arena_value(name, v, num_envs):
    """a table argument as float64: [3] (batch-wide) or [num_envs, 3] (per environment); ValueError on any other shape, a non-finite
    or a non-positive value"""
    import torch

    a = np.array(v.detach().cpu() if torch.is_tensor(v) else v, dtype=np.float64)
    if a.shape not in ((3,), (num_envs, 3)):
        raise ValueError("{} must be a length-3 sequence or a [num_envs, 3] = [{}, 3] array, got shape {}".format(name, num_envs, a.shape))
    if not (np.all(np.isfinite(a)) and np.all(a > 0)):
        raise ValueError("{} must be finite and > 0, got {}".format(name, v))
    return a


def table_model(model, table_offset, full_size, friction):
    """a copy of `model` with the reference's table of `full_size` / `friction` and the robot base behind it (the rules above); the
    table geom's bounding data and the model's derived constants come from the compiler's own code"""
    import copy

    from ..mjcf.compiler import GEOM_BOX, _set_const, primitive_geom_props

    m = copy.copy(model)
    for f in ("body_pos", "geom_size", "geom_friction", "geom_rbound", "geom_aabb"):
        setattr(m, f, np.array(getattr(model, f), dtype=np.float64))
    g, tb, rb = m.names["geom"].index(TABLE_GEOM), m.names["body"].index(TABLE_BODY), m.names["body"].index(ROBOT_ROOT)
    m.body_pos[tb] = [table_offset[0], table_offset[1], table_offset[2] - full_size[2] / 2]
    m.geom_size[g] = np.asarray(full_size, dtype=np.float64) / 2
    m.geom_friction[g] = friction
    _, _, m.geom_rbound[g], m.geom_aabb[g] = primitive_geom_props(GEOM_BOX, m.geom_size[g])
    m.body_pos[rb, 0] = -0.16 - full_size[0] / 2
    _set_const(m)
    return m


class BatchedMujocoEnv(ContactQueries):
    """N copies of one task on one GPU.  All returned arrays are torch.cuda tensors with leading dim N.
    contact_queries=True switches the contact export on (BatchedSim.set_contact_export) before the first reset, so that
    check_contact / get_contacts / _check_grasp (envs/contacts.py) can read the contacts of the last substep.  data_queries=True
    does the same for the step-1 arrays (BatchedSim.set_step1_export), so that sim.data (robosuite_b200/data.py) reads the poses,
    Jacobians and mass matrices of the last substep.  dynamics_queries=True switches on the step-2 export
    (BatchedSim.set_step2_export) and the contact export, so that sim.data reads the actuator, smooth and constraint forces, the
    constraint rows and the per-contact forces (sim.data.contact_force()) of the last substep.
    placement_initializer: a robosuite_b200.placement_samplers UniformRandomSampler or SequentialCompositeSampler naming the task's
    objects; every reset then places them by the reference's rules on the device (see _setup_placement).  None: the task's default
    placement."""

    maxcon = None  # per-environment contact / constraint-row capacity (None: engine defaults 32 / 64); overflow sets warn bit 4
    maxefc = None
    # capacities of the tail kernel's small tier (contacts, rows): what all but ~0.1 % of this task's environment-substeps stay within
    # under random actions (measured: tools/probe_instr.py); None = no tiering
    tier_small = None
    # per-environment tensors of the task layer that a snapshot carries besides the engine rows, the episode clocks and `done`
    # (attribute names; [N, ...] device tensors)
    _task_state = ()
    # the reference's table arguments and their defaults (Lift, Stack, NutAssembly); a task whose table cannot take other values
    # names the reason in `_table_args_refused`, and non-default values raise NotImplementedError with it
    table_full_size_default = (0.8, 0.8, 0.05)
    table_friction_default = (1.0, 5e-3, 1e-4)
    _table_args_refused = None

    def __init__(self, robots="Panda", num_envs=1, device=0, controller_configs=None, control_freq=20, horizon=500,
                 ignore_done=False, reward_scale=1.0, reward_shaping=False, use_object_obs=True, seed=None,
                 initialization_noise="default", precision="f32", xml=None, has_renderer=False,
                 has_offscreen_renderer=False, use_camera_obs=False, hard_reset=False, lite_physics=True, model=None,
                 kernel_mode="pipeline", sim_cls=None, contact_queries=False, data_queries=False,
                 dynamics_queries=False, placement_initializer=None, table_full_size=None, table_friction=None, **kwargs):
        """table_full_size / table_friction: the reference's TableArena arguments (see table_model), a length-3 sequence for every
        environment (the model is edited before the engine is created) or a [num_envs, 3] array or tensor, one table per environment
        (per-environment geom values and a moved table and robot base on the device; set_table changes them later)"""
        import torch

        if has_renderer or has_offscreen_renderer or use_camera_obs:
            raise NotImplementedError("rendering / camera observations are out of scope of the batched engine")
        if not lite_physics:
            raise NotImplementedError("only lite_physics=True semantics (environments/base.py:494-503) are implemented")
        self.robot_name = robots if isinstance(robots, str) else robots[0]
        self.num_envs = int(num_envs)
        self.control_freq = control_freq
        self.horizon = horizon
        self.ignore_done = ignore_done
        self.reward_scale = reward_scale
        self.reward_shaping = reward_shaping
        self.hard_reset = hard_reset
        self.use_object_obs = use_object_obs
        self.initialization_noise = {"magnitude": 0.02, "type": "gaussian"} if initialization_noise == "default" \
            else (initialization_noise or {"magnitude": 0.0, "type": "gaussian"})
        self.model = model if model is not None else self._load_model(xml)
        self.model = self._arena_model(self.model)
        per_env_table = self._table_arguments(table_full_size, table_friction)
        self.model_timestep = self.model.opt_timestep
        self.control_timestep = 1.0 / control_freq
        if control_freq <= 0:
            raise ValueError("Control frequency {} is invalid".format(control_freq))
        self.n_substeps = int(self.control_timestep / self.model_timestep)
        caps = {k: v for k, v in (("maxcon", kwargs.get("maxcon", self.maxcon)), ("maxefc", kwargs.get("maxefc", self.maxefc)),
                                  ("tier_small", kwargs.get("tier_small", self.tier_small))) if v}
        # sim_cls: test hook (tests/oracle_sim.py drives the same host code on the CPU oracle); the product path is BatchedSim
        self.sim = (sim_cls or BatchedSim)(self.model, self.num_envs, device=device, precision=precision, **caps)
        self.device = self.sim.torch_device
        self.dtype = self.sim.dtype
        self.composite_controller_config = cc.load_composite_controller_config(controller_configs, self.robot_name)
        self.gripper_type = "panda" if self.robot_name == "Panda" else "rethink"
        self._ctrl_cfg = cc.resolve(self.model, self.composite_controller_config, CtrlCfg, gripper=self.gripper_type)
        self.sim.ctrl_config(self._ctrl_cfg)
        self._setup_references()
        ob = ObsBuilder()
        self._setup_observables(ob)
        op, a, b, self._obs_slices, self._modality_slices = ob.tables()
        self._obs_op = op
        self._obs_mods = {}  # observable name -> {"sampling_rate": Hz, "corruptor": spec or None} (modify_observable)
        self.obs_dim = len(op)
        self.sim.obs_config(op, a, b)
        self._setup_task()
        self._table_ov = None
        if per_env_table:
            self._setup_table_overrides()
        self.sim.set_export(False)
        self._contact_queries = bool(contact_queries or dynamics_queries)  # contact_force() reads the contact records too
        if self._contact_queries:
            self.sim.set_contact_export(True)
        if data_queries:
            self.sim.set_step1_export(True)
        if dynamics_queries:
            self.sim.set_step2_export(True)
        # "pipeline": phase kernels + global collision work lists (fastest in steady state); "fused": one kernel per step
        self.sim.set_mode(1 if kernel_mode == "pipeline" else 0)
        self.rng = torch.Generator(device=self.device)
        self.seed = seed
        if seed is not None:
            self.rng.manual_seed(int(seed))
        self.placement_initializer = placement_initializer
        if placement_initializer is not None:
            self._setup_placement()
        self.timestep = torch.zeros(self.num_envs, dtype=torch.long, device=self.device)
        self.done = torch.zeros(self.num_envs, dtype=torch.bool, device=self.device)
        self.cur_time = 0.0
        self._max_steps_since_reset = 0  # host-side upper bound of `timestep` (avoids a device sync per step)
        self._host_steps = np.zeros(self.num_envs, dtype=np.int64)  # host mirror of `timestep` (None once a caller resets by device mask)
        self.reset()

    # ---- to be provided by tasks
    def _load_model(self, xml):
        raise NotImplementedError

    def _setup_references(self):
        m = self.model
        jn = m.names["joint"]
        pf = "robot0_"
        self.robot_joints = [i for i, n in enumerate(jn) if n and n.startswith(pf) and int(m.jnt_type[i]) == 3]
        self._ref_joint_pos_indexes = [int(m.jnt_qposadr[j]) for j in self.robot_joints]
        self._ref_joint_vel_indexes = [int(m.jnt_dofadr[j]) for j in self.robot_joints]
        self.gripper_joints = [i for i, n in enumerate(jn) if n and n.startswith("gripper0_")]
        self._ref_gripper_joint_pos_indexes = [int(m.jnt_qposadr[j]) for j in self.gripper_joints]
        self._ref_gripper_joint_vel_indexes = [int(m.jnt_dofadr[j]) for j in self.gripper_joints]
        self.eef_site_id = m.names["site"].index("gripper0_right_grip_site")
        self.eef_body_id = m.names["body"].index("robot0_right_hand")

    def _setup_observables(self, ob):
        """robot proprio observables in the reference's order (robots/robot.py:347-392, 412-484)"""
        mod = "robot0_proprio"
        qp, qv = self._ref_joint_pos_indexes, self._ref_joint_vel_indexes
        ob.add("robot0_joint_pos", mod, [(OB_QPOS, i, 0) for i in qp])
        ob.add("robot0_joint_pos_cos", mod, [(OB_COS_QPOS, i, 0) for i in qp])
        ob.add("robot0_joint_pos_sin", mod, [(OB_SIN_QPOS, i, 0) for i in qp])
        ob.add("robot0_joint_vel", mod, [(OB_QVEL, i, 0) for i in qv])
        ob.add("robot0_joint_acc", mod, [(OB_QACC, i, 0) for i in qv])
        ob.add("robot0_eef_pos", mod, [(OB_SITE_POS, self.eef_site_id, k) for k in range(3)])
        ob.add("robot0_eef_quat", mod, [(OB_BODY_QUAT_XYZW, self.eef_body_id, k) for k in range(4)])
        ob.add("robot0_eef_quat_site", mod, [(OB_SITE_QUAT_XYZW, self.eef_site_id, k) for k in range(4)])
        ob.add("robot0_gripper_qpos", mod, [(OB_QPOS, i, 0) for i in self._ref_gripper_joint_pos_indexes])
        ob.add("robot0_gripper_qvel", mod, [(OB_QVEL, i, 0) for i in self._ref_gripper_joint_vel_indexes])

    def _setup_task(self):
        pass

    def _arena_model(self, model):
        """the task's arena arguments other than the table applied to the model (PickPlace's bins); the default: none"""
        return model

    # ---- the table arguments (TableArena: see table_model)
    def _table_arguments(self, full_size, friction):
        """validate table_full_size / table_friction, apply batch-wide values that differ from the defaults to self.model, and
        return whether any value is per environment.  Default values leave the model untouched."""
        size = None if full_size is None else _arena_value("table_full_size", full_size, self.num_envs)
        fric = None if friction is None else _arena_value("table_friction", friction, self.num_envs)
        default = [v is None or (v.ndim == 1 and np.array_equal(v, d))
                   for v, d in ((size, self.table_full_size_default), (fric, self.table_friction_default))]
        if self._table_args_refused is not None and not all(default):
            raise NotImplementedError("{}: table_full_size / table_friction: {}".format(type(self).__name__, self._table_args_refused))
        self.table_full_size = np.array(self.table_full_size_default if size is None else size)
        self.table_friction = np.array(self.table_friction_default if fric is None else fric)
        batch = [v is not None and v.ndim == 1 and not dflt for v, dflt in zip((size, fric), default)]
        if any(batch):
            self.model = table_model(self.model, self.table_offset, self.table_full_size if batch[0] else self.table_full_size_default,
                                     self.table_friction if batch[1] else self.table_friction_default)
        return any(v is not None and v.ndim == 2 for v in (size, fric))

    def _setup_table_overrides(self):
        """per-environment table: size and friction of table_collision through the engine's model overrides, the table body and the
        robot's welded root through pose overrides (the root's welded subtree follows it), written by set_table"""
        m, sim = self.model, self.sim
        g, tb, rb = m.names["geom"].index(TABLE_GEOM), m.names["body"].index(TABLE_BODY), m.names["body"].index(ROBOT_ROOT)
        self._table_ov = (sim.model_override("geom_size", g), sim.model_override("geom_friction", g),
                          sim.body_pose_override_tree(tb)[0], sim.body_pose_override_tree(rb)[0])
        self.set_table(self.table_full_size, self.table_friction)

    def set_table(self, full_size=None, friction=None, mask=None):
        """Give the masked environments (bool [num_envs] device tensor, None = all) a new table: full_size / friction as a length-3
        sequence or a [num_envs, 3] array or tensor (rows of unmasked environments are ignored), None = unchanged.  Needs a handle
        built with per-environment table arguments.  The table, its friction and the robot base move at once and the derived
        constants are recomputed; meant to be followed by reset(mask=mask).  Called mid-episode, the next step starts from the old
        state in the new scene: a cube resting on a thinner table falls onto it, and the arm, carried with its base, keeps its joint
        angles."""
        import torch

        if self._table_ov is None:
            raise RuntimeError("set_table needs per-environment table arguments at construction: table_full_size / table_friction "
                               "as a [num_envs, 3] array")
        size_ov, fric_ov, table_pos, base_pos = self._table_ov
        sel = torch.ones(self.num_envs, dtype=torch.bool) if mask is None else mask.detach().to("cpu", torch.bool).reshape(self.num_envs)
        rows = sel.numpy()

        def per_env(name, v):
            a = _arena_value(name, v, self.num_envs)
            return np.broadcast_to(a, (self.num_envs, 3)).copy()

        def put(dst, src):
            dst[sel.to(dst.device)] = torch.as_tensor(src[rows], device=dst.device, dtype=dst.dtype)

        size = per_env("table_full_size", full_size) if full_size is not None else None
        fric = per_env("table_friction", friction) if friction is not None else None
        if size is not None:
            off = self.table_offset
            put(size_ov, size / 2)
            put(table_pos, np.stack([np.full(self.num_envs, float(off[0])), np.full(self.num_envs, float(off[1])),
                                     off[2] - size[:, 2] / 2], 1))
            base = base_pos.detach().cpu().numpy().astype(np.float64)
            base[:, 0] = -0.16 - size[:, 0] / 2
            put(base_pos, base)
            self.table_full_size = np.broadcast_to(self.table_full_size, (self.num_envs, 3)).copy()
            self.table_full_size[rows] = size[rows]
        if fric is not None:
            put(fric_ov, fric)
            self.table_friction = np.broadcast_to(self.table_friction, (self.num_envs, 3)).copy()
            self.table_friction[rows] = fric[rows]
        self._table_mask8 = None if mask is None else sel.to(device=self.device, dtype=torch.uint8).contiguous()  # kept alive
        self.sim.set_const(self._table_mask8)

    def _robot_reset_qpos(self, n):
        """[n, nq] float64 qpos0 with the arm at init_qpos + noise and the gripper at its init pose
        (robots/robot.py:247-259, gripper init_qpos)"""
        import torch

        from .lift import GRIPPER_INIT_QPOS, PANDA_INIT_QPOS, SAWYER_INIT_QPOS

        dev = self.device
        q = self._dev_const("qpos0", self.model.qpos0).repeat(n, 1)
        init = PANDA_INIT_QPOS if self.robot_name == "Panda" else SAWYER_INIT_QPOS
        mag = float(self.initialization_noise["magnitude"])
        if self.initialization_noise["type"] == "gaussian":
            noise = torch.randn((n, len(init)), generator=self.rng, device=dev, dtype=torch.float64) * mag
        else:
            noise = (torch.rand((n, len(init)), generator=self.rng, device=dev, dtype=torch.float64) * 2 - 1) * mag
        q[:, self._dev_index("arm_qpos", self._ref_joint_pos_indexes)] = self._dev_const("arm_init", init) + noise
        q[:, self._dev_index("grip_qpos", self._ref_gripper_joint_pos_indexes)] = self._dev_const("grip_init", GRIPPER_INIT_QPOS[self.robot_name])
        return q

    def _dev_const(self, key, value, dtype=None):
        """device-resident copy of a host constant, uploaded once (the reset path must not touch the host: it runs inside step())"""
        import torch

        c = self.__dict__.setdefault("_dev_consts", {})
        if key not in c:
            c[key] = torch.as_tensor(np.asarray(value), device=self.device, dtype=dtype or torch.float64)
        return c[key]

    def _dev_index(self, key, idx):
        import torch

        return self._dev_const("idx_" + key, np.asarray(idx, dtype=np.int64), dtype=torch.long)

    @staticmethod
    def _place_free_body(q, adr, x, y, z, yaw):
        """free-joint qpos <- position + rotation about z"""
        import torch

        q[:, adr] = x
        q[:, adr + 1] = y
        q[:, adr + 2] = z
        q[:, adr + 3] = torch.cos(yaw / 2)
        q[:, adr + 4] = 0
        q[:, adr + 5] = 0
        q[:, adr + 6] = torch.sin(yaw / 2)

    def _sample_reset_state(self, n):
        raise NotImplementedError

    def _placement_objects(self):
        """the task's objects for a placement_initializer: name -> dict(radius, bottom, top, qpos_adr, body) (lower() in
        placement_samplers.py), in the order the reference's _load_model adds them; None: the task takes no sampler"""
        return None

    def _setup_placement(self):
        """what the reference's _load_model does with a given sampler: reset() and add_objects(the task's objects) for a single
        sampler; a SequentialCompositeSampler keeps the objects its samplers name (its reset() would drop them).  The program is
        lowered once and configured on the handle; the Philox key comes from make(seed=...) under a tag of its own."""
        from ..placement_samplers import SequentialCompositeSampler, lower

        objects = self._placement_objects()
        if objects is None:
            raise NotImplementedError("{} does not take a placement_initializer".format(type(self).__name__))
        sampler = self.placement_initializer
        if not isinstance(sampler, SequentialCompositeSampler):
            sampler.reset()
            sampler.add_objects(list(objects))
        self._placement_names, entries = lower(sampler, objects)
        self.sim.place_config(entries)
        self._place_seed = self._tagged_seed(0x504C4143)  # "PLAC"
        self._place_counter = 0

    def _place_objects(self, q):
        """the sampler's placements of the environments being reset (the mask reset() was given) in one launch: free joints into q
        (float64 [N, nq], before any parking), world-welded bodies into their pose overrides.  The counter advances on the host."""
        import torch

        mask = self._reset_mask_arg
        self._place_mask8 = None if mask is None else mask.to(device=self.device, dtype=torch.uint8).contiguous()  # kept alive
        self.sim.place_objects(q, self._place_mask8, self._place_seed, self._place_counter)
        self._place_counter = (self._place_counter + 1) & 0xFFFFFFFF

    def _tagged_seed(self, tag):
        """a 64-bit key derived from make(seed=...) (a seed drawn once when seed is None) and a tag of the stream's own"""
        base = int(self.seed) if self.seed is not None else int(np.random.SeedSequence().generate_state(1, np.uint64)[0])
        return int(np.random.SeedSequence([base & (2 ** 64 - 1), tag]).generate_state(1, np.uint64)[0])

    def _randomize_model(self, mask):
        """per-reset draws that live outside qpos, applied to the masked environments before the engine's reset: placements the
        reference writes into MODEL constants (Door: door.py:417-427) and the drawn object of single_object_mode 1 (PickPlace,
        NutAssembly); mask: bool [N] on the device or None"""

    def reward(self, action=None):
        raise NotImplementedError

    def _check_success(self):
        raise NotImplementedError

    # ---- API
    @property
    def action_dim(self):
        return int(self._ctrl_cfg.action_dim)

    @property
    def action_spec(self):
        """(low, high) bounds (robot_env.py:271-285): the arm controller's control_limits, then the gripper's [-1, 1].  The arm's
        are its input limits (od entries: 6 for OSC_POSE, 3 for OSC_POSITION, n_arm for the joint-space kinds), preceded in the
        variable impedance modes by the gain limits: [damping_ratio_min, kp_min, input_min] in "variable", [kp_min, input_min] in
        "variable_kp" (d entries each: 6 for OSC, n_arm for JOINT_POSITION)"""
        c = self._ctrl_cfg
        if c.kind in (2, 3, 4):  # joint-space controllers: per-joint input limits
            od = d = c.n_arm
            low, high = list(c.jv_in_min)[:od], list(c.jv_in_max)[:od]
        else:
            od, d = (3 if c.kind == 5 else 6), 6
            low, high = list(c.input_min)[:od], list(c.input_max)[:od]
        mode = getattr(c, "impedance_mode", 0)
        if mode == 2:
            low, high = list(c.kp_min)[:d] + low, list(c.kp_max)[:d] + high
        elif mode == 1:
            low = list(c.damping_ratio_min)[:d] + list(c.kp_min)[:d] + low
            high = list(c.damping_ratio_max)[:d] + list(c.kp_max)[:d] + high
        n = c.action_dim - len(low)
        return np.array(low + [-1.0] * n), np.array(high + [1.0] * n)

    def _fingerpad_geoms(self):
        """left / right fingerpad geom id lists (models/grippers/*_gripper.py `_important_geoms`)"""
        gn = self.model.names["geom"]
        if self.gripper_type == "panda":
            l, r = ["gripper0_right_finger1_pad_collision"], ["gripper0_right_finger2_pad_collision"]
        else:
            l, r = ["gripper0_right_l_fingerpad_g0"], ["gripper0_right_r_fingerpad_g0"]
        return [gn.index(x) for x in l], [gn.index(x) for x in r]

    def reset(self, mask=None, host_mask=None):
        """Re-initialise all (or masked) environments: robot init pose + noise, gripper open, task objects sampled,
        controllers rebuilt (goal <- current eef pose), observations force-updated (environments/base.py:277-347).
        Everything runs on the device without a host round trip: an initial state is sampled for every environment (a few small
        tensor ops) and `b2s_reset_envs` applies it to the masked ones, so a per-step auto-reset costs three short launches.
        host_mask: the same mask as a numpy bool array when the caller has it (keeps the host mirror of the episode clocks exact)."""
        import torch

        # the two hooks run in this order, both over all num_envs rows: _randomize_model applies to the masked environments what
        # _sample_reset_state drew besides qpos (single_object_mode 1 hands its object draw over in `_sel_draw`, envs/single_object.py)
        self._reset_mask_arg = mask  # the environments a placement_initializer places (_place_objects)
        q = self._sample_reset_state(self.num_envs).to(self.dtype).contiguous()
        self._randomize_model(None if mask is None else mask.to(device=self.device).bool())
        if mask is None:
            self.timestep.zero_()
            self.done.zero_()
            self._max_steps_since_reset = 0
            self._host_steps = np.zeros(self.num_envs, dtype=np.int64)
            self.sim.reset_envs(None, q)
        else:
            self._reset_mask8 = mask.to(device=self.device, dtype=torch.uint8).contiguous()  # a copy (the caller may pass `self.done`), kept alive
            mask = self._reset_mask8.bool()
            self.timestep.masked_fill_(mask, 0)
            self.done.masked_fill_(mask, False)
            self.sim.reset_envs(self._reset_mask8, q)
            if host_mask is not None and self._host_steps is not None:
                self._host_steps[np.asarray(host_mask, dtype=bool)] = 0
                self._max_steps_since_reset = int(self._host_steps.max())
            else:
                self._host_steps = None  # episode clocks now only known on the device; `_max_steps_since_reset` stays an upper bound
        self._reset_qpos = q
        self.cur_time = 0.0
        return self._get_observations()

    def set_episode_steps(self, steps):
        """Set the per-environment episode clocks (e.g. to stagger the episode phases of a long-running vector environment)."""
        import torch

        h = np.asarray(steps.cpu() if torch.is_tensor(steps) else steps, dtype=np.int64).reshape(self.num_envs)
        self._host_steps = h.copy()
        self.timestep[:] = torch.as_tensor(h, device=self.device)
        self._max_steps_since_reset = int(h.max())

    def host_done(self):
        """numpy bool [N]: which environments have reached the horizon, from the host mirror of the episode clocks; None if unknown"""
        if self._host_steps is None or self.ignore_done:
            return None
        return self._host_steps >= self.horizon

    def reset_to(self, qpos, qvel=None):
        """Put every environment into the given state and do what reset() does afterwards (forward, controllers rebuilt,
        observation cache emptied and force-updated): `set_state` + the tail of environments/base.py:277-347.
        qpos: [nq] or [N, nq]"""
        import torch

        def dev(x):
            return x.to(device=self.device, dtype=self.dtype) if torch.is_tensor(x) else torch.as_tensor(np.asarray(x), dtype=self.dtype, device=self.device)

        q = dev(qpos)
        self.sim.qpos[:] = q if q.ndim == 2 else q.unsqueeze(0).expand(self.num_envs, -1)
        if qvel is None:
            self.sim.qvel[:] = 0
        else:
            v = dev(qvel)
            self.sim.qvel[:] = v if v.ndim == 2 else v.unsqueeze(0).expand(self.num_envs, -1)
        self.sim.qacc[:] = 0
        self.sim.qacc_warmstart[:] = 0
        self.sim.ctrl[:] = 0
        self.sim.time[:] = 0
        self.timestep[:] = 0
        self.done[:] = False
        self.sim.obs_fresh[:] = 1
        self.sim.warn[:] = 0
        self._max_steps_since_reset = 0
        self._host_steps = np.zeros(self.num_envs, dtype=np.int64)
        self.sim.forward()
        self.sim.ctrl_reset(None)
        self.cur_time = 0.0
        return self._get_observations()

    def step(self, action):
        """One control step = n_substeps x {step1, controller, step2} in one kernel launch (base.py:467-521)."""
        import torch

        # an env can only be done once the longest-running one has reached the horizon: no device sync before that
        if not self.ignore_done and self._max_steps_since_reset >= self.horizon:
            hd = self.host_done()
            if bool(hd.any()) if hd is not None else bool(self.done.any()):
                raise ValueError("executing action in terminated episode")
        self._max_steps_since_reset += 1
        if self._host_steps is not None:
            self._host_steps += 1
        action = torch.as_tensor(action, dtype=self.dtype, device=self.device).contiguous()
        assert action.shape == (self.num_envs, self.action_dim), "environment got invalid action dimension -- expected {}, got {}".format(
            (self.num_envs, self.action_dim), tuple(action.shape))
        self.timestep += 1
        self.sim.env_step(action, self.n_substeps)
        self.cur_time += self.control_timestep
        reward = self.reward(action)
        self.done = (self.timestep >= self.horizon) & (not self.ignore_done)
        # (an environment whose state diverged was reset to the model defaults by the engine, like mj_resetData after mj_checkPos / Vel / Acc;
        # as in the reference the episode simply continues from there - info["sim_warn"] bit 32 tells the caller)
        # per-environment engine flags since the last reset, as a device tensor (no host sync here; see SIM_WARN_BITS): a non-zero entry means
        # the episode is no longer a faithful MuJoCo rollout (capacity overflow, singular mass matrix / Hessian, diverged state)
        return self._get_observations(), reward, self.done, {"sim_warn": self.sim.warn}

    # ---- observable modifiers (utils/observables.py Observable.set_sampling_rate / set_corrupter, MujocoEnv.modify_observable)
    _UNSUPPORTED_OBS_ATTRS = {
        "delayer": "observation delays are not implemented",
        "filter": "observation filters are not implemented",
        "sensor": "sensors are fixed observation-table programs on the device",
        "enabled": "enabling or disabling an observable changes obs_dim",
        "active": "activating or deactivating an observable changes obs_dim",
    }

    def modify_observable(self, observable_name, attribute, modifier):
        """Change one observable of every environment (environments/base.py modify_observable): attribute "corruptor" (or the
        reference's spelling "corrupter") takes a spec from robosuite_b200.observables (create_gaussian_noise_corruptor /
        create_uniform_noise_corruptor) or None (no noise); "sampling_rate" takes a rate in Hz > 0.  Sampling and noise run on the
        device after every substep, as the reference's Observable.update does (delay 0).  The noise key is derived from
        make(seed=...) (a seed drawn once when seed is None) under a tag of its own, so the same seed given to
        BatchedDomainRandomizationWrapper draws an independent stream.  Nothing changes if the call raises.  A handle whose
        observables all keep the control rate and no corruptor runs the unmodified path."""
        import math

        from ..observables import GaussianNoiseCorruptor, UniformNoiseCorruptor

        if observable_name not in self._obs_slices:
            raise ValueError("No valid observable with name {} found. Options are: {}".format(observable_name, list(self._obs_slices)))
        if attribute in self._UNSUPPORTED_OBS_ATTRS:
            raise NotImplementedError("modify_observable: attribute {!r}: {}".format(attribute, self._UNSUPPORTED_OBS_ATTRS[attribute]))
        cur = dict(self._obs_mods.get(observable_name, {"sampling_rate": float(self.control_freq), "corruptor": None}))
        if attribute in ("corruptor", "corrupter"):
            if modifier is not None and not isinstance(modifier, (GaussianNoiseCorruptor, UniformNoiseCorruptor)):
                raise NotImplementedError("modify_observable: attribute {!r}: arbitrary callables cannot run on the device; "
                                          "use robosuite_b200.observables.create_gaussian_noise_corruptor / "
                                          "create_uniform_noise_corruptor".format(attribute))
            cur["corruptor"] = modifier
        elif attribute == "sampling_rate":
            a, b = self._obs_slices[observable_name]
            if any(int(op) in (OB_REL_POS_LAG, OB_REL_QUAT_LAG) for op in self._obs_op[a:b]):
                raise NotImplementedError("modify_observable: attribute 'sampling_rate' of {}: the reference computes it from a hidden "
                                          "gripper-pose observable that keeps the control rate".format(observable_name))
            rate = float(modifier)
            if not (math.isfinite(rate) and rate > 0):
                raise ValueError("sampling_rate must be a finite rate in Hz > 0, got {}".format(modifier))
            cur["sampling_rate"] = rate
        else:
            raise ValueError("Invalid observable attribute specified. Requested: {}, valid options are {}".format(
                attribute, ["sensor", "corrupter", "filter", "delayer", "sampling_rate", "enabled", "active"]))
        mods = dict(self._obs_mods)
        mods[observable_name] = cur
        self._upload_obs_modifiers(mods)  # raises before anything is changed on the device
        self._obs_mods = mods

    def _upload_obs_modifiers(self, obs_mods):
        """the device tables of `obs_mods` (name -> rate / corruptor), one observable per slice of _obs_slices in observation order"""
        from ..engine import CORRUPT_NONE

        names = list(self._obs_slices)
        mods = [obs_mods.get(n, {"sampling_rate": float(self.control_freq), "corruptor": None}) for n in names]
        if all(m["corruptor"] is None and m["sampling_rate"] == float(self.control_freq) for m in mods):
            self.sim.obs_modifiers([], [])  # the default rule: every sample on the last substep, no noise
            return
        if len(names) > 32:
            raise NotImplementedError("observable modifiers support at most 32 observables ({} has {})".format(type(self).__name__, len(names)))
        row_obs = np.zeros(self.obs_dim, dtype=np.int32)
        for o, n in enumerate(names):
            a, b = self._obs_slices[n]
            row_obs[a:b] = o
        spec = [(1.0 / m["sampling_rate"],) + (m["corruptor"].spec() if m["corruptor"] is not None else (CORRUPT_NONE, 0.0, 0.0, -np.inf, np.inf))
                for m in mods]
        if "_obs_noise_seed" not in self.__dict__:
            # "OBSN": the observation-noise stream of this seed (Philox keys of the dynamics perturbation take the seed itself)
            self._obs_noise_seed = self._tagged_seed(0x4F42534E)
        self.sim.obs_modifiers(row_obs, spec, self._obs_noise_seed)

    def check_sim_warnings(self):
        """Host-side check of the engine flags (one device sync): raises SimulationError naming the flags and how many
        environments carry them.  The reference surfaces the same conditions as mujoco warnings / MujocoException."""
        from ..errors import SimulationError

        w = self.sim.warn
        if bool((w != 0).any()):
            bits = {name: int(((w & bit) != 0).sum()) for bit, name in SIM_WARN_BITS.items()}
            raise SimulationError("engine flags raised: " + ", ".join(f"{k} in {v} envs" for k, v in bits.items() if v))

    def _get_observations(self):
        """OrderedDict of per-observable tensors plus the per-modality concatenations (base.py:429-465)."""
        obs = self.sim.obs
        out = OrderedDict()
        for name, (a, b) in self._obs_slices.items():
            out[name] = obs[:, a:b]
        for name, (a, b) in self._modality_slices.items():
            out[name] = obs[:, a:b]
        return out

    def flat_obs(self):
        """[N, obs_dim] tensor aliasing the kernel's observation buffer (GymWrapper-style flattening)"""
        return self.sim.obs

    def get_state(self):
        return self.sim.get_state()

    # ---- whole-environment snapshots: engine rows (BatchedSim.snapshot) + the episode clocks, `done` and the task's tensors
    def get_env_state(self, env_ids=None):
        """Everything that decides the next control steps of environments `env_ids` (host indices, None = all in order), for
        set_env_state / clone_envs / state_io.save_snapshot(extra=state["tensors"]).  Not included: `rng` and the domain-randomisation
        counter, which belong to the handle, not to an environment; later draws stay keyed by the destination's index."""
        import torch

        idx = None if env_ids is None else np.asarray(env_ids.cpu() if torch.is_tensor(env_ids) else env_ids, dtype=np.int64).reshape(-1)
        sel = slice(None) if idx is None else torch.as_tensor(idx, device=self.device)
        tensors = {name: getattr(self, name)[sel].clone() for name in ("timestep", "done") + tuple(self._task_state)}
        host = None if self._host_steps is None else self._host_steps[slice(None) if idx is None else idx].copy()
        return {"sim": self.sim.snapshot(idx), "tensors": tensors, "host_steps": host, "max_steps": int(self._max_steps_since_reset)}

    def set_env_state(self, state, src=None):
        """Environment e takes entry src[e] of `state` (get_env_state; -1 keeps it, None: entry e).  src on the host (list / numpy)
        keeps the host mirror of the episode clocks exact, so BatchedGymWrapper resets a restored environment on its source's
        schedule; a device tensor (e.g. an argmax) avoids a host round trip, and the mirror becomes unknown as after a device-mask
        reset.  An index out of range leaves its environment untouched and sets warn bit 256.  No physics runs: observations and task
        outputs are the source's; the exported derived arrays follow at the next step."""
        import torch

        k = len(state["sim"])
        self.sim.restore(state["sim"], src)
        if src is None:
            for name, t in state["tensors"].items():
                getattr(self, name).copy_(t)
            on_device = False
            h = np.arange(self.num_envs)
        else:
            on_device = torch.is_tensor(src) and src.is_cuda
            g = src.to(device=self.device, dtype=torch.long) if on_device else torch.as_tensor(
                np.asarray(src.cpu() if torch.is_tensor(src) else src, dtype=np.int64), device=self.device)
            ok = (g >= 0) & (g < k)
            g = g.clamp(0, max(k - 1, 0))
            for name, t in state["tensors"].items():
                dst = getattr(self, name)
                dst.copy_(torch.where(ok.view((-1,) + (1,) * (dst.ndim - 1)), t.to(dst.device)[g], dst))
            h = None if on_device else np.asarray(src.cpu() if torch.is_tensor(src) else src, dtype=np.int64).reshape(self.num_envs)
        if on_device or self._host_steps is None or state["host_steps"] is None:
            self._host_steps = None  # `_max_steps_since_reset` stays an upper bound of every clock
            self._max_steps_since_reset = max(self._max_steps_since_reset, int(state["max_steps"]))
        else:
            ok_h = (h >= 0) & (h < k)
            self._host_steps[ok_h] = np.asarray(state["host_steps"])[h[ok_h]]
            self._max_steps_since_reset = int(self._host_steps.max())
        return self._get_observations()

    def clone_envs(self, src):
        """environment e continues from the current state of environment src[e] (-1 keeps its own): get_env_state + set_env_state"""
        return self.set_env_state(self.get_env_state(), src)

    def close(self):
        self.sim.close()
