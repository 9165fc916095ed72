"""Batched counterpart of robosuite's GymWrapper (robosuite/wrappers/gym_wrapper.py:26-180).

Same key selection and flattening rule (`object-state` first, then `robot{i}_proprio-state`), same 5-tuple `step` return,
but every array carries a leading environment axis and lives on the GPU, and finished episodes are reset inside `step`
(gymnasium VectorEnv "next-step autoreset is too late for a fused simulator": the observation returned for a finished
environment is the first observation of its next episode, the final one is in `info["final_observation"]`).  `step` never
synchronises with the device: which episodes ended is known on the host (horizon-only termination) and the masked reset is a
device-side launch sequence (`b2s_reset_envs`).

BatchedDomainRandomizationWrapper is the dynamics part of robosuite's DomainRandomizationWrapper
(robosuite/wrappers/domain_randomization_wrapper.py) on per-environment model values perturbed on the device."""
import numpy as np


class _Box:
    """duck-typed stand-in for gymnasium.spaces.Box (bounds, shape, dtype, contains, sample) when gymnasium is not installed"""

    def __init__(self, low, high, dtype=np.float32):
        self.low, self.high = np.asarray(low, dtype=dtype), np.asarray(high, dtype=dtype)
        self.shape, self.dtype = self.low.shape, np.dtype(dtype)

    def contains(self, x):
        x = np.asarray(x)
        return x.shape == self.shape and bool(np.all(x >= self.low) and np.all(x <= self.high))

    def sample(self, rng=None):
        rng = rng or np.random.default_rng()
        lo, hi = np.where(np.isfinite(self.low), self.low, -1.0), np.where(np.isfinite(self.high), self.high, 1.0)
        return rng.uniform(lo, hi).astype(self.dtype)

    def __repr__(self):
        return f"Box({self.low.min()}, {self.high.max()}, {self.shape}, {self.dtype})"


def _make_spaces(obs_dim, act_low, act_high, num_envs):
    """(single_observation_space, single_action_space, observation_space, action_space) as in gym_wrapper.py:70-85, batched like a
    gymnasium VectorEnv; real gymnasium spaces when the package is importable"""
    hi = np.full((obs_dim,), np.inf, dtype=np.float32)
    try:
        from gymnasium import spaces
        from gymnasium.vector.utils import batch_space

        so, sa = spaces.Box(-hi, hi, dtype=np.float32), spaces.Box(act_low, act_high, dtype=np.float32)
        return so, sa, batch_space(so, num_envs), batch_space(sa, num_envs)
    except ImportError:
        so, sa = _Box(-hi, hi), _Box(act_low, act_high)
        rep = lambda b: _Box(np.tile(b.low, (num_envs, 1)), np.tile(b.high, (num_envs, 1)))
        return so, sa, rep(so), rep(sa)


class BatchedGymWrapper:
    def __init__(self, env, keys=None, flatten_obs=True, auto_reset=True):
        self.env = env
        self.name = env.robot_name + "_" + type(env).__name__.replace("Batched", "")
        self.reward_range = (0, env.reward_scale)
        if keys is None:  # gym_wrapper.py:52-61
            keys = []
            if env.use_object_obs:
                keys += ["object-state"]
            keys += ["robot0_proprio-state"]
        self.keys = keys
        self.flatten_obs = flatten_obs
        self.auto_reset = auto_reset
        self.num_envs = env.num_envs
        obs = env._get_observations()
        self.obs_dim = int(sum(obs[k].shape[1] for k in self.keys if k in obs))
        low, high = env.action_spec
        self.action_low, self.action_high = np.asarray(low, dtype=np.float32), np.asarray(high, dtype=np.float32)
        self.single_observation_shape = (self.obs_dim,)
        self.single_action_shape = self.action_low.shape
        # gymnasium VectorEnv surface (gym_wrapper.py:70-85 per environment, batched along the leading axis)
        (self.single_observation_space, self.single_action_space, self.observation_space,
         self.action_space) = _make_spaces(self.obs_dim, self.action_low, self.action_high, self.num_envs)
        self.metadata, self.render_mode, self.spec = {"autoreset_mode": "same_step"}, None, None

    def __getattr__(self, name):  # the environment's own API (modify_observable, get_env_state, ...), as robosuite's Wrapper delegates
        if name == "env":
            raise AttributeError(name)
        return getattr(self.env, name)

    def _flatten_obs(self, obs_dict):
        import torch

        return torch.cat([obs_dict[k].reshape(self.num_envs, -1) for k in self.keys if k in obs_dict], dim=1)

    def _filter_obs(self, obs_dict):
        return {k: obs_dict[k] for k in self.keys if k in obs_dict}

    def _format(self, obs_dict):
        return self._flatten_obs(obs_dict) if self.flatten_obs else self._filter_obs(obs_dict)

    def reset(self, seed=None, options=None):
        if seed is not None:
            if not isinstance(seed, int):
                raise TypeError("Seed must be an integer type!")
            self.env.rng.manual_seed(seed)
        return self._format(self.env.reset()), {}

    def step(self, action):
        """-> (obs, reward [N], terminated [N] bool, truncated [N] bool, info).  `terminated` is the reference's `done`
        (horizon reached, environments/base.py:513-514); the reference never truncates."""
        import torch

        ob_dict, reward, done, info = self.env.step(action)
        obs = self._format(ob_dict)
        terminated = done.clone()
        env = self.env
        if self.auto_reset and not env.ignore_done and env._max_steps_since_reset >= env.horizon:
            # the horizon is the only termination rule (environments/base.py:513-514), so the host mirror of the episode clocks says which
            # environments finished without reading `done` back; the reset itself is a masked device-side launch sequence.  Without the mirror
            # (a caller reset by device mask) the masked reset is enqueued anyway: it is a no-op for an all-false mask
            hd = env.host_done()
            if hd is None or hd.any():
                info = dict(info)
                info["final_observation"] = obs.clone() if self.flatten_obs else {k: v.clone() for k, v in obs.items()}
                info["sim_warn"] = info["sim_warn"].clone()  # the reset clears the flags of the finished episodes
                obs = self._format(env.reset(mask=done, host_mask=hd))
        return obs, reward, terminated, torch.zeros_like(terminated), info

    def get_env_state(self, env_ids=None):
        return self.env.get_env_state(env_ids)

    def set_env_state(self, state, src=None):
        """restore environments (BatchedMujocoEnv.set_env_state) -> the formatted observation.  A restored environment is auto-reset
        on its source's schedule: exactly through the host mirror of the clocks for host-given `src`, by device mask otherwise."""
        return self._format(self.env.set_env_state(state, src))

    def clone_envs(self, src):
        return self._format(self.env.clone_envs(src))

    def compute_reward(self, achieved_goal=None, desired_goal=None, info=None):
        return self.env.reward()

    def close(self):
        self.env.close()


# the reference's DEFAULT_DYNAMICS_ARGS (wrappers/domain_randomization_wrapper.py) under the same names.  The knobs the batched engine
# cannot honour default to False here and raise NotImplementedError when set: local body poses (randomize_position /
# randomize_quaternion), joint stiffness (shared by the batch: the engine's springs are not per environment), and the global density / viscosity.
DEFAULT_DYNAMICS_ARGS = {
    "randomize_density": False, "randomize_viscosity": False,
    "density_perturbation_ratio": 0.1, "viscosity_perturbation_ratio": 0.1,
    "body_names": None, "randomize_position": False, "randomize_quaternion": False, "randomize_inertia": True, "randomize_mass": True,
    "position_perturbation_size": 0.0015, "quaternion_perturbation_size": 0.003,
    "inertia_perturbation_ratio": 0.02, "mass_perturbation_ratio": 0.02,
    "geom_names": None, "randomize_friction": True, "randomize_solref": True, "randomize_solimp": True,
    "friction_perturbation_ratio": 0.1, "solref_perturbation_ratio": 0.1, "solimp_perturbation_ratio": 0.1,
    "joint_names": None, "randomize_stiffness": False, "randomize_frictionloss": True, "randomize_damping": True,
    "randomize_armature": True, "stiffness_perturbation_ratio": 0.1, "frictionloss_perturbation_size": 0.05,
    "damping_perturbation_size": 0.01, "armature_perturbation_size": 0.01,
}
_UNSUPPORTED_DYNAMICS = ("randomize_position", "randomize_quaternion", "randomize_stiffness", "randomize_density", "randomize_viscosity")
_MAX_OBJECTS = 8  # per-handle cap of per-environment geoms, and separately bodies (b2s_model_override)


class BatchedDomainRandomizationWrapper:
    """Dynamics-only counterpart of the reference's DomainRandomizationWrapper (wrappers/domain_randomization_wrapper.py) for a
    batched environment: every environment draws its own masses, moments, friction, solref / solimp, joint damping, armature and
    friction loss around the model's values, on the device (b2s_perturb_model: one launch per randomisation, no host data).

    - reset(mask, host_mask) perturbs the masked environments, then resets them; the reset recomputes their derived constants.
    - step(action) perturbs, before stepping, every environment whose own episode clock is a multiple of randomize_every_n_steps (the
      reference's per-episode step counter; 0 = never) and recomputes its derived constants.  The mask is computed on the device.
    - Every randomisation call advances a counter; draws are Philox4x32-10 keyed by the seed, so an environment's values depend only on
      (seed, counter, environment index).
    Attributes are delegated to `env`, so BatchedGymWrapper(BatchedDomainRandomizationWrapper(env)) auto-resets (and so randomises)
    exactly the finished environments.

    Defaults that differ from the reference: body_names=None selects the task's free objects (the moving bodies outside the robot and
    gripper; Door: its door and latch), geom_names=None the colliding primitive geoms of those bodies plus the two fingerpads, and
    joint_names=None every dof.  A selection of more than 8 geoms or 8 bodies raises NotImplementedError: name the objects.  Each dof
    draws its own value (a free joint's six dofs draw six)."""

    def __init__(self, env, seed=None, randomize_dynamics=True, dynamics_randomization_args=None, randomize_on_reset=True,
                 randomize_every_n_steps=1, randomize_color=False, randomize_camera=False, randomize_lighting=False):
        for knob, on in (("randomize_color", randomize_color), ("randomize_camera", randomize_camera),
                         ("randomize_lighting", randomize_lighting)):
            if on:
                raise NotImplementedError(f"{knob}: the batched engine has no renderer")
        args = dict(DEFAULT_DYNAMICS_ARGS)
        unknown = set(dynamics_randomization_args or {}) - set(args)
        if unknown:
            raise ValueError("unknown dynamics randomization arguments: %s" % sorted(unknown))
        args.update(dynamics_randomization_args or {})
        for knob in _UNSUPPORTED_DYNAMICS:
            if args[knob]:
                raise NotImplementedError(f"{knob}: the batched engine cannot randomise this per environment (set it to False)")
        if int(randomize_every_n_steps) < 0:
            raise ValueError("randomize_every_n_steps must be >= 0")
        self.env = env
        self.randomize_dynamics = bool(randomize_dynamics)
        self.randomize_on_reset = bool(randomize_on_reset)
        self.randomize_every_n_steps = int(randomize_every_n_steps)
        self.dynamics_randomization_args = args
        self.seed = int(np.random.SeedSequence().entropy & (2 ** 64 - 1)) if seed is None else int(seed) & (2 ** 64 - 1)
        self.counter = 0
        self.perturb_spec = self._build_spec(args) if self.randomize_dynamics else []
        self._mask8 = None
        sim = env.sim
        for field, oid, *_ in self.perturb_spec:
            sim.model_override(field, None if oid < 0 or field.startswith("dof_") else oid)
        sim.perturb_config(self.perturb_spec)

    def __getattr__(self, name):  # only called for attributes the wrapper does not have itself
        if name == "env":
            raise AttributeError(name)
        return getattr(self.env, name)

    # ---- selection
    def _ids(self, kind, names):
        table = self.env.model.names[kind]
        try:
            return [table.index(n) for n in names]
        except ValueError as e:
            raise ValueError(f"unknown {kind} name: {e}") from None

    def default_bodies(self):
        """the task's free objects: moving bodies outside the robot and the gripper"""
        m = self.env.model
        bn = m.names["body"]
        return [b for b in range(1, m.nbody) if int(m.body_weldid[b]) != 0 and not bn[b].startswith(("robot0_", "gripper0_"))]

    def default_geoms(self, bodies):
        """the colliding sphere / capsule / ellipsoid / cylinder / box geoms of `bodies`, then the two fingerpads"""
        m = self.env.model
        colliding = {int(g) for p in m.pair_geom for g in p}
        own = [g for g in range(m.ngeom) if int(m.geom_bodyid[g]) in bodies and g in colliding and int(m.geom_type[g]) in (2, 3, 4, 5, 6)]
        left, right = self.env._fingerpad_geoms()
        return own + [g for g in left + right if g not in own]

    def _build_spec(self, a):
        """perturb_config entries (field, id, mode, amplitude, one_draw) of the selected objects"""
        env, m = self.env, self.env.model
        spec = []
        body_on = a["randomize_mass"] or a["randomize_inertia"]
        geom_on = a["randomize_friction"] or a["randomize_solref"] or a["randomize_solimp"]
        bodies = self.default_bodies() if a["body_names"] is None else self._ids("body", a["body_names"])
        if body_on:
            if len(bodies) > _MAX_OBJECTS:
                raise NotImplementedError("%d bodies selected, the engine holds %d per-environment bodies: pass body_names"
                                          % (len(bodies), _MAX_OBJECTS))
            drawn = {env.cube_body_id} if getattr(env, "_cube_ov", None) is not None else set()
            clash = [m.names["body"][b] for b in bodies if b in drawn]
            if clash:
                raise ValueError("the task draws the mass and inertia of %s itself (per_env_cube_size): leave it out of body_names or "
                                 "switch off randomize_mass / randomize_inertia" % clash)
            for b in bodies:
                if a["randomize_mass"]:
                    spec.append(("body_mass", b, "scale", a["mass_perturbation_ratio"], False))
                if a["randomize_inertia"]:  # one factor for the three moments keeps the triangle inequality
                    spec.append(("body_inertia", b, "scale", a["inertia_perturbation_ratio"], True))
        if geom_on:
            geoms = self.default_geoms(bodies) if a["geom_names"] is None else self._ids("geom", a["geom_names"])
            if getattr(env, "_table_ov", None) is not None and m.names["geom"].index("table_collision") in geoms:
                raise ValueError("the task sets the friction of table_collision itself (per-environment table_friction / "
                                 "table_full_size, set_table): leave it out of geom_names")
            if len(geoms) > _MAX_OBJECTS:
                raise NotImplementedError("%d geoms selected, the engine holds %d per-environment geoms: pass geom_names"
                                          % (len(geoms), _MAX_OBJECTS))
            for g in geoms:
                for knob, field, ratio in (("randomize_friction", "geom_friction", "friction_perturbation_ratio"),
                                           ("randomize_solref", "geom_solref", "solref_perturbation_ratio"),
                                           ("randomize_solimp", "geom_solimp", "solimp_perturbation_ratio")):
                    if a[knob]:
                        spec.append((field, g, "scale", a[ratio], False))
        if a["joint_names"] is None:
            dofs = [-1]
        else:
            dofs = []
            for j in self._ids("joint", a["joint_names"]):
                adr, n = int(m.jnt_dofadr[j]), {0: 6, 1: 3}.get(int(m.jnt_type[j]), 1)
                dofs += list(range(adr, adr + n))
        for knob, field, size in (("randomize_damping", "dof_damping", "damping_perturbation_size"),
                                  ("randomize_armature", "dof_armature", "armature_perturbation_size"),
                                  ("randomize_frictionloss", "dof_frictionloss", "frictionloss_perturbation_size")):
            if a[knob]:
                spec += [(field, d, "shift", a[size], False) for d in dofs]
        return spec

    # ---- randomisation
    def randomize_domain(self, mask=None):
        """perturb the masked environments (bool / uint8 [N] device mask, None = all) around the model's values; the derived
        constants follow at the next set_const or reset"""
        import torch

        if not self.perturb_spec:
            return
        if mask is not None:
            self._mask8 = mask.to(device=self.env.device, dtype=torch.uint8).contiguous()  # kept alive until the next call
        self.env.sim.perturb_model(None if mask is None else self._mask8, seed=self.seed, counter=self.counter)
        self.counter += 1

    def reset(self, mask=None, host_mask=None):
        if self.randomize_on_reset:
            self.randomize_domain(mask)
        return self.env.reset(mask=mask, host_mask=host_mask)

    def step(self, action):
        if self.perturb_spec and self.randomize_every_n_steps > 0:
            due = (self.env.timestep % self.randomize_every_n_steps) == 0  # per-environment episode clock, on the device
            self.randomize_domain(due)
            self.env.sim.set_const(self._mask8)
        return self.env.step(action)
