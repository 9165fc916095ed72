"""Observable sampling rates and corruptors on the host: the sampling rule (tests/observable_ref.py), the CPU oracle's substep loop,
the environment API on the oracle and every argument check.  The device is covered by tests/test_gpu_observables.py."""
import math

import numpy as np
import pytest
import torch

from robosuite_b200.engine import CORRUPT_GAUSSIAN, CORRUPT_NONE, CORRUPT_UNIFORM, B2SError
from robosuite_b200.observables import create_gaussian_noise_corruptor, create_uniform_noise_corruptor
from tests.observable_ref import corrupt, noise_uniforms, sample_substeps
from tests.util import load

DT = 0.002


def test_the_control_rate_samples_on_the_last_substep():
    """20 Hz with dt 0.002: one sample per control step, after substep 25 - the instant the default path samples at"""
    assert load("Lift_Panda").opt_timestep == DT
    assert sample_substeps(20, DT, 25, 200) == [[25]] * 200


@pytest.mark.parametrize("rate, table", [
    (10, [[], [25]] * 4),
    (40, [[13, 25]] * 8),
    # T = 71.43 dt: the period closes after substeps 21, 17, 14 ... of every third control step (fmod keeps the remainder)
    (7, [[], [], [22], [], [], [18], [], [], [15], [], []]),
    (500, [list(range(1, 26))] * 8),
])
def test_sample_instants(rate, table):
    assert sample_substeps(rate, DT, 25, len(table)) == table


def test_the_noise_restatement():
    """draws depend on (seed, env, count, row) only; Gaussian and uniform arithmetic as documented, clipping exact"""
    u1, u2 = noise_uniforms(7, 3, 5, [0, 1, 2])
    a1, a2 = noise_uniforms(7, 3, 5, [2])
    assert u1[2] == a1[0] and u2[2] == a2[0]
    assert np.all((u1 >= 0) & (u1 < 1)) and len(set(u1)) == 3
    assert not np.array_equal(noise_uniforms(7, 3, 6, [0])[0], u1[:1]) and not np.array_equal(noise_uniforms(8, 3, 5, [0])[0], u1[:1])
    v = np.array([1.0, 2.0, 3.0])
    g = corrupt(v, (0.05, CORRUPT_GAUSSIAN, 0.5, 2.0, -math.inf, math.inf), 7, 3, 5, [0, 1, 2])
    assert np.array_equal(g, v + (0.5 + 2.0 * (np.sqrt(-2.0 * np.log(1.0 - u1)) * np.cos(2.0 * np.pi * u2))))
    un = corrupt(v, (0.05, CORRUPT_UNIFORM, -0.1, 0.3, -math.inf, math.inf), 7, 3, 5, [0, 1, 2])
    assert np.array_equal(un, v + (-0.1 + 0.4 * u1))
    c = corrupt(v, (0.05, CORRUPT_UNIFORM, 5.0, 6.0, 1.5, 2.5), 7, 3, 5, [0, 1, 2])
    assert np.array_equal(c, [2.5, 2.5, 2.5])
    assert np.array_equal(corrupt(v, (0.05, CORRUPT_NONE, 9, 9, 0, 0), 7, 3, 5, [0, 1, 2]), v)


def _make(task="Lift", n=2, sim_cls=None, **kw):
    import robosuite_b200 as suite
    from tests.oracle_sim_observables import ObsOracleSim

    return suite.make(task, robots="Panda", num_envs=n, seed=0, sim_cls=sim_cls or ObsOracleSim, precision="f64", **kw)


def test_the_substep_loop_is_the_oracle_env_step():
    """without modifiers the substep-by-substep loop reproduces o_env_step bit for bit"""
    from tests.oracle_sim import OracleSim

    a, b = _make(sim_cls=OracleSim), _make()
    act = torch.as_tensor(np.random.default_rng(0).uniform(-1, 1, (3, 2, a.action_dim)))
    for k in range(3):
        oa, _, _, _ = a.step(act[k])
        ob, _, _, _ = b.step(act[k])
        assert torch.equal(a.sim.qpos, b.sim.qpos) and torch.equal(a.sim.qvel, b.sim.qvel) and torch.equal(a.sim.obs, b.sim.obs)


def test_env_api_with_modifiers_on_the_oracle():
    env = _make()
    env.modify_observable("cube_pos", "corruptor", create_gaussian_noise_corruptor(0.0, 0.01))
    env.modify_observable("robot0_joint_pos", "sampling_rate", 10)
    env.modify_observable("gripper_to_cube_pos", "corruptor", create_uniform_noise_corruptor(-0.1, 0.1, low=-0.05, high=0.05))
    sim = env.sim
    assert sim.obs_timer.shape == (2, len(env._obs_slices)) and torch.all(sim.obs_nsample == 0)
    o0 = env.reset()
    names = list(env._obs_slices)
    ic, ij = names.index("cube_pos"), names.index("robot0_joint_pos")
    assert torch.all(sim.obs_nsample == 1)
    cube = torch.as_tensor(np.stack([o.xpos[env.cube_body_id] for o in sim.o]))
    assert not torch.equal(o0["cube_pos"], cube) and torch.allclose(o0["cube_pos"], cube, atol=0.1)
    assert torch.all(o0["gripper_to_cube_pos"].abs() <= 0.05)
    jp0 = o0["robot0_joint_pos"].clone()
    act = torch.zeros((2, env.action_dim), dtype=torch.float64)
    o1, _, _, _ = env.step(act)
    assert torch.equal(o1["robot0_joint_pos"], jp0)  # 10 Hz: no sample in the first control step
    assert torch.all(sim.obs_nsample[:, ij] == 1) and torch.all(sim.obs_nsample[:, ic] == 2)
    o2, _, _, _ = env.step(act)
    assert not torch.equal(o2["robot0_joint_pos"], jp0) and torch.all(sim.obs_nsample[:, ij] == 2)
    # a masked reset forces a sample and restarts the timers; the counts continue
    env.reset(mask=torch.tensor([True, False]))
    assert sim.obs_nsample[0, ij] == 3 and sim.obs_nsample[1, ij] == 2
    assert sim.obs_timer[0, ij] == DT
    # back to the defaults: the handle returns to the unmodified path
    env.modify_observable("cube_pos", "corruptor", None)
    env.modify_observable("robot0_joint_pos", "sampling_rate", 20)
    env.modify_observable("gripper_to_cube_pos", "corruptor", None)
    assert sim._mods is None


def test_modify_observable_reaches_through_the_gym_wrapper():
    from robosuite_b200.wrappers import BatchedGymWrapper

    env = BatchedGymWrapper(_make())
    env.modify_observable("cube_quat", "sampling_rate", 40)
    assert env.env.sim._mods is not None


def test_unsupported_attributes_and_bad_arguments():
    env = _make("NutAssemblyRound", n=1)
    for attr in ("delayer", "filter", "sensor", "enabled", "active"):
        with pytest.raises(NotImplementedError, match=attr):
            env.modify_observable("robot0_joint_pos", attr, None)
    with pytest.raises(NotImplementedError, match="callable"):
        env.modify_observable("robot0_joint_pos", "corruptor", lambda x: x)
    lag = [n for n in env._obs_slices if n.endswith("_to_robot0_eef_pos")]
    assert lag
    with pytest.raises(NotImplementedError, match="sampling_rate"):
        env.modify_observable(lag[0], "sampling_rate", 10)
    env.modify_observable(lag[0], "corruptor", create_gaussian_noise_corruptor(0.0, 0.1))  # corruptors are fine there
    with pytest.raises(ValueError):
        env.modify_observable("no_such_observable", "corruptor", None)
    with pytest.raises(ValueError):
        env.modify_observable("robot0_joint_pos", "no_such_attribute", None)
    for bad in (0, -5, math.inf, math.nan):
        with pytest.raises(ValueError):
            env.modify_observable("robot0_joint_pos", "sampling_rate", bad)
    with pytest.raises(ValueError):
        create_gaussian_noise_corruptor(0.0, -1.0)
    with pytest.raises(ValueError):
        create_gaussian_noise_corruptor(math.nan, 1.0)
    with pytest.raises(ValueError):
        create_uniform_noise_corruptor(0.2, 0.1)
    with pytest.raises(ValueError):
        create_uniform_noise_corruptor(0.0, 0.1, low=1.0, high=0.0)


def test_library_argument_checks_on_the_oracle():
    """the checks of b2s_obs_modifiers, restated by the CPU stand-in (the device raises on the same cases: test_gpu_observables)"""
    from tests.oracle_sim_observables import ObsOracleSim

    sim = ObsOracleSim(load("Lift_Panda"), 1)
    ok = (0.05, CORRUPT_GAUSSIAN, 0.0, 0.1, -1.0, 1.0)
    with pytest.raises(B2SError, match="not configured"):
        sim.obs_modifiers([0], [ok])
    sim.obs_config([0, 0], [0, 1], [0, 0])
    for mods in ([ok] * 33,
                 [(0.0,) + ok[1:]], [(-1.0,) + ok[1:]], [(math.inf,) + ok[1:]], [(math.nan,) + ok[1:]],
                 [(0.05, 7, 0, 0, 0, 0)],
                 [(0.05, CORRUPT_GAUSSIAN, 0.0, -0.1, -1.0, 1.0)],
                 [(0.05, CORRUPT_GAUSSIAN, math.nan, 0.1, -1.0, 1.0)],
                 [(0.05, CORRUPT_UNIFORM, 0.2, 0.1, -1.0, 1.0)],
                 [(0.05, CORRUPT_UNIFORM, 0.0, 0.1, 1.0, -1.0)]):
        with pytest.raises(B2SError):
            sim.obs_modifiers([0, 0], mods)
    with pytest.raises(B2SError, match="out of range"):
        sim.obs_modifiers([0, 1], [ok])
    with pytest.raises(B2SError, match="out of range"):
        sim.obs_modifiers([0, -1], [ok, ok])
    sim.obs_modifiers([0, 1], [ok, ok])
    sim.obs_modifiers([], [])


def test_the_lagged_quaternion_normalises_a_corrupted_cache():
    """with modifiers, `{obj}_to_robot0_eef_quat` builds the cached pose with the reference's quat2mat: a scaled cache gives the
    unit-cache value, a zero cache the identity"""
    from scipy.spatial.transform import Rotation

    from robosuite_b200.envs.base import OB_REL_QUAT_LAG
    from tests.observable_ref import quat2mat
    from tests.oracle_sim import _q2m

    q = Rotation.random(random_state=3).as_quat()  # xyzw
    assert np.allclose(quat2mat(q), _q2m(q[[3, 0, 1, 2]]), atol=1e-15) and np.allclose(quat2mat(2.5 * q), quat2mat(q), atol=1e-15)
    assert np.array_equal(quat2mat(np.zeros(4)), np.identity(3))
    env = _make("NutAssemblyRound", n=1)
    obj = [n[: -len("_to_robot0_eef_quat")] for n in env._obs_slices if n.endswith("_to_robot0_eef_quat")][0]
    a0 = env._obs_slices[obj + "_to_robot0_eef_quat"][0]
    qs = env._obs_slices[obj + "_quat"][0]
    op, a, b = (int(x[a0]) for x in env.sim._obs_tab)
    assert op == OB_REL_QUAT_LAG
    env.modify_observable(obj + "_quat", "corruptor", create_gaussian_noise_corruptor(0.0, 0.01))
    sim, o = env.sim, env.sim.o[0]
    prev = np.zeros(env.obs_dim)
    vals = {}
    for scale in (1.0, 1.3, 0.0):
        prev[qs:qs + 4] = scale * q
        vals[scale] = np.array([sim._value(o, op, a, (b & ~255) | k, prev, False) for k in range(4)])
    assert np.allclose(vals[1.3], vals[1.0], atol=1e-14)
    hand = _q2m(o.xquat[(b >> 16) & 255])
    expect = Rotation.from_matrix(hand.T).as_quat()
    assert np.allclose(vals[0.0], expect if expect[3] >= 0 else -expect, atol=1e-14)


def test_modify_observable_spellings_rollback_and_noise_key():
    from robosuite_b200.engine import B2SError

    env = _make()
    env.modify_observable("cube_pos", "corrupter", create_gaussian_noise_corruptor(0.0, 0.01))  # the reference's spelling
    assert env._obs_mods["cube_pos"]["corruptor"] is not None and env.sim._mods is not None
    # independent of a dynamics perturbation keyed by the same make(seed=...)
    other = _make()
    other.modify_observable("cube_pos", "corruptor", create_gaussian_noise_corruptor(0.0, 0.01))
    assert env._obs_noise_seed != env.seed and env._obs_noise_seed == other._obs_noise_seed
    before = {k: dict(v) for k, v in env._obs_mods.items()}
    seed_before = env.sim._mods

    def boom(*a, **k):
        raise B2SError("refused")

    env.sim.obs_modifiers = boom
    with pytest.raises(B2SError):
        env.modify_observable("cube_quat", "sampling_rate", 40)
    assert env._obs_mods == before and env.sim._mods is seed_before
