"""Observable sampling rates and corruptors on the device (b2s_obs_modifiers, BatchedMujocoEnv.modify_observable): the unmodified path
is untouched, the device follows the CPU oracle with the restated rule and draws, the lagged observables read the corrupted cache,
the noise has its distribution, the three schedules agree bit for bit, and snapshots / resets carry or restart the timers."""
import math

import numpy as np
import pytest

from robosuite_b200.engine import CORRUPT_GAUSSIAN, CORRUPT_NONE, CORRUPT_UNIFORM
from robosuite_b200.observables import create_gaussian_noise_corruptor, create_uniform_noise_corruptor
from tests.schedules import make_env, random_actions, run

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

RATES = (20, 10, 40, 7)


def _configure(env, zero=False):
    """mixed rates and corruptors over the environment's observables (the lagged ones keep the control rate)"""
    from robosuite_b200.envs.base import OB_REL_POS_LAG, OB_REL_QUAT_LAG

    for k, name in enumerate(env._obs_slices):
        a, b = env._obs_slices[name]
        lag = any(int(op) in (OB_REL_POS_LAG, OB_REL_QUAT_LAG) for op in env._obs_op[a:b])
        if zero:
            env.modify_observable(name, "corruptor", create_gaussian_noise_corruptor(0.0, 0.0))
            continue
        if not lag:
            env.modify_observable(name, "sampling_rate", RATES[k % len(RATES)])
        if k % 3 == 0:
            env.modify_observable(name, "corruptor", create_gaussian_noise_corruptor(0.001, 0.01, low=-2.0, high=2.0))
        elif k % 3 == 1:
            env.modify_observable(name, "corruptor", create_uniform_noise_corruptor(-0.02, 0.01, low=-0.5, high=0.5))


def _masked_run(env, acts, split):
    r = run(env, acts[:split])
    mask = torch.zeros(env.num_envs, dtype=torch.bool, device=env.device)
    mask[::3] = True
    env.reset(mask=mask)
    return r + run(env, acts[split:])


@pytest.mark.parametrize("prec", ["f64", "f32"])
def test_without_modifiers_nothing_changes(prec):
    """a handle that configured and cleared modifiers, and one with zero-amplitude noise at the control rate, are bit-identical
    to a handle that never configured them"""
    n = 32
    envs = [make_env("Lift", n, 1, 4, precision=prec) for _ in range(3)]
    _configure(envs[1])
    for name in envs[1]._obs_slices:
        envs[1].modify_observable(name, "sampling_rate", 20)
        envs[1].modify_observable(name, "corruptor", None)
    _configure(envs[2], zero=True)
    assert envs[2].sim.array("obs_timer").shape[1] == len(envs[2]._obs_slices)
    for e in envs:
        e.reset()
    acts = random_actions(envs[0], 6)
    res = [_masked_run(e, acts, 3) for e in envs]
    for r in res[1:]:
        for x, y in zip(res[0], r):
            assert torch.equal(x, y)
    for e in envs:
        e.close()


def _oracle_pair(task, prec, n=4):
    """the same task on the device and on the CPU oracle, both reset to the same states (tests/test_gpu_dynamics_override.py)"""
    import robosuite_b200 as suite
    from tests.oracle_sim_observables import ObsOracleSim
    from tests.test_gpu_dynamics_override import _task_model_and_states

    m, q = _task_model_and_states(task, n)
    kw = {"door_placement": (0.08, 0.0, -np.pi / 2 - 0.125)} if task == "Door" else {}
    out = []
    for sim_cls, p in ((None, prec), (ObsOracleSim, "f64")):
        env = suite.make(task, robots="Panda", num_envs=n, seed=11, model=m, precision=p, sim_cls=sim_cls, **kw)
        qt = torch.as_tensor(q, device=env.device)
        env._sample_reset_state = lambda k, qt=qt: qt.clone()
        out.append(env)
    return out


@pytest.mark.parametrize("task", ["Lift", "Stack", "Door"])
@pytest.mark.parametrize("prec", ["f64", "f32"])
def test_device_follows_the_oracle(task, prec):
    dev, ref = _oracle_pair(task, prec)
    for env in (dev, ref):
        _configure(env)
        env.reset()
    n = dev.num_envs
    gen = np.random.default_rng(2)
    acts = gen.uniform(-0.2, 0.2, (9, n, dev.action_dim))
    worst = worst_q = 0.0
    for t in range(9):
        if t == 4:
            mask = np.array([e % 2 == 1 for e in range(n)])
            for env in (dev, ref):
                env.reset(mask=torch.as_tensor(mask, device=env.device))
        od, _, _, _ = dev.step(torch.as_tensor(acts[t], device=dev.device, dtype=dev.dtype))
        orf, _, _, _ = ref.step(torch.as_tensor(acts[t], dtype=torch.float64))
        a, b = dev.sim.obs.double().cpu().numpy(), ref.sim.obs.numpy()
        worst = max(worst, float(np.max(np.abs(a - b) / np.maximum(1.0, np.abs(b)))))
        worst_q = max(worst_q, float(np.max(np.abs(dev.sim.qpos.double().cpu().numpy() - ref.sim.qpos.numpy()))))
        assert np.array_equal(dev.sim.obs_nsample.cpu().numpy(), ref.sim.obs_nsample.numpy()), t
        assert np.array_equal(dev.sim.obs_sampled.cpu().numpy(), ref.sim.obs_sampled.numpy()), t
    # the sample instants, flags and counts agree exactly (above); the values carry the engine-vs-oracle difference of the trajectory
    # itself (the OSC controller under actions: measured 3.4e-7 on Lift f64, with qpos), so the draws are checked bit for bit by
    # test_draws_match_the_restatement against the device's own exported poses
    print(task, prec, "obs vs oracle with modifiers: max error %.3g (qpos %.3g)" % (worst, worst_q))
    assert worst <= (1e-5 if prec == "f64" else 1e-3)
    assert int(dev.sim.warn.abs().max()) == 0
    dev.close()


@pytest.mark.parametrize("prec", ["f64", "f32"])
def test_draws_match_the_restatement(prec):
    """pose observables sampled on the last substep, against tests/observable_ref.corrupt of the exported poses of that substep:
    f64 to the ulps of log / cos / sqrt, f32 to its rounding; the counts (noise counters) follow the host rule"""
    import robosuite_b200 as suite
    from tests.observable_ref import corrupt

    env = suite.make("Lift", robots="Panda", num_envs=64, seed=8, precision=prec, kernel_mode="fused")
    env.modify_observable("cube_pos", "corruptor", create_gaussian_noise_corruptor(0.01, 0.02, low=-10.0, high=0.84))
    env.modify_observable("cube_quat", "corruptor", create_uniform_noise_corruptor(-0.01, 0.03))
    env.modify_observable("cube_quat", "sampling_rate", 40)
    env.sim.set_export(True)
    env.reset()
    mods = {n: ((1.0 / 20 if n == "cube_pos" else 1.0 / 40),) + env._obs_mods[n]["corruptor"].spec() for n in ("cube_pos", "cube_quat")}
    seed = env._obs_noise_seed
    tol = 1e-12 if prec == "f64" else 1e-6
    acts = random_actions(env, 4)
    b = env.cube_body_id
    for t in range(4):
        env.step(acts[t])
        torch.cuda.synchronize()
        cnt = env.sim.obs_nsample.cpu().numpy()
        clean = {"cube_pos": env.sim.xpos[:, b].double().cpu().numpy(), "cube_quat": env.sim.xquat[:, b][:, [1, 2, 3, 0]].double().cpu().numpy()}
        names = list(env._obs_slices)
        for name, m in mods.items():
            a0, a1 = env._obs_slices[name]
            got = env.sim.obs[:, a0:a1].double().cpu().numpy()
            o = names.index(name)
            for e in range(env.num_envs):
                ref = corrupt(clean[name][e], m, seed, e, int(cnt[e, o]) - 1, range(a0, a1))
                assert np.max(np.abs(got[e] - ref)) <= tol, (name, t, e)
        assert np.all(cnt[:, names.index("cube_pos")] == 2 + t) and np.all(cnt[:, names.index("cube_quat")] == 3 + 2 * t)
    env.close()


def test_noise_reaches_the_lagged_observables():
    """`{obj}_to_robot0_eef_pos` reads the corrupted `{obj}_pos` of the previous sample: R_hand^T (cache - eef site)"""
    import robosuite_b200 as suite

    env = suite.make("NutAssemblyRound", robots="Panda", num_envs=8, seed=1, precision="f64", kernel_mode="fused")
    obj = [n[: -len("_to_robot0_eef_pos")] for n in env._obs_slices if n.endswith("_to_robot0_eef_pos")][0]
    env.modify_observable(obj + "_pos", "corruptor", create_gaussian_noise_corruptor(0.0, 0.05))
    env.sim.set_export(True)
    env.reset()
    acts = random_actions(env, 3)
    for t in range(3):
        prev = env.sim.obs[:, slice(*env._obs_slices[obj + "_pos"])].clone()
        obs, _, _, _ = env.step(acts[t])
        torch.cuda.synchronize()
        site = env.sim.site_xpos[:, env.eef_site_id]
        q = env.sim.xquat[:, env.eef_body_id]
        w, x, y, z = q.unbind(-1)
        R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                         2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                         2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1).view(-1, 3, 3)
        expect = torch.einsum("eji,ej->ei", R, prev - site)
        assert torch.allclose(obs[obj + "_to_robot0_eef_pos"], expect, atol=1e-12, rtol=0), t
        # the noise is in it: the noise-free cache would give another value
        true_pos = env.sim.xpos[:, env.obj_body_id[obj]]
        assert float((prev - true_pos).abs().max()) > 1e-3 or t == 0
    env.close()


@pytest.mark.parametrize("zero", [False, True])
def test_corrupted_quaternions_reach_the_lagged_observables_normalised(zero):
    """`{obj}_to_robot0_eef_quat` from a corrupted (not unit) `{obj}_quat` cache: R_hand^T quat2mat(cache) with the reference's
    normalising quat2mat (tests/observable_ref.quat2mat), the identity for a cache clipped to zero"""
    from scipy.spatial.transform import Rotation

    import robosuite_b200 as suite
    from tests.observable_ref import quat2mat

    env = suite.make("NutAssemblyRound", robots="Panda", num_envs=8, seed=1, precision="f64", kernel_mode="fused")
    obj = [n[: -len("_to_robot0_eef_quat")] for n in env._obs_slices if n.endswith("_to_robot0_eef_quat")][0]
    corr = create_uniform_noise_corruptor(0.0, 0.0, low=0.0, high=0.0) if zero else create_gaussian_noise_corruptor(0.0, 0.05)
    env.modify_observable(obj + "_quat", "corruptor", corr)
    env.sim.set_export(True)
    env.reset()
    acts = random_actions(env, 3)
    for t in range(3):
        prev = env.sim.obs[:, slice(*env._obs_slices[obj + "_quat"])].double().cpu().numpy()
        obs, _, _, _ = env.step(acts[t])
        torch.cuda.synchronize()
        hand = env.sim.xquat[:, env.eef_body_id].double().cpu().numpy()
        got = obs[obj + "_to_robot0_eef_quat"].double().cpu().numpy()
        for e in range(env.num_envs):
            assert zero == (not prev[e].any())
            Re = Rotation.from_quat(hand[e][[1, 2, 3, 0]]).as_matrix()
            q = Rotation.from_matrix(Re.T @ quat2mat(prev[e])).as_quat()
            q = -q if q[3] < 0 else q
            assert np.allclose(got[e], q, atol=1e-9, rtol=0), (t, e, got[e], q)
        assert zero or np.abs(np.linalg.norm(prev, axis=1) - 1.0).max() > 1e-2  # the cache really is not unit-length
    env.close()


def test_noise_statistics_bounds_and_clipping():
    import robosuite_b200 as suite

    n = 4096
    env = suite.make("Lift", robots="Panda", num_envs=n, seed=3, precision="f64")
    env.modify_observable("cube_pos", "corruptor", create_gaussian_noise_corruptor(0.01, 0.02))
    env.modify_observable("cube_quat", "corruptor", create_uniform_noise_corruptor(-0.01, 0.03))
    env.modify_observable("gripper_to_cube_pos", "corruptor", create_gaussian_noise_corruptor(0.0, 1.0, low=-0.05, high=0.05))
    env.sim.set_export(True)
    obs = env.reset()
    torch.cuda.synchronize()
    b, s = env.cube_body_id, env.eef_site_id
    d = (obs["cube_pos"] - env.sim.xpos[:, b]).flatten()
    se = 0.02 / math.sqrt(d.numel())
    assert abs(float(d.mean()) - 0.01) < 5 * se
    assert abs(float(d.std()) - 0.02) < 5 * 0.02 / math.sqrt(2 * d.numel())
    xq = env.sim.xquat[:, b][:, [1, 2, 3, 0]]
    u = (obs["cube_quat"] - xq).flatten()
    assert float(u.min()) >= -0.01 - 1e-15 and float(u.max()) < 0.03 + 1e-15
    assert abs(float(u.mean()) - 0.01) < 5 * (0.04 / math.sqrt(12)) / math.sqrt(u.numel())
    g = obs["gripper_to_cube_pos"]
    assert float(g.min()) == -0.05 and float(g.max()) == 0.05
    assert int((g.abs() == 0.05).sum()) > g.numel() // 2
    env.close()


@pytest.mark.parametrize("tier", [None, (4, 16)])
def test_schedules_agree_with_modifiers(tier):
    """fused, pipeline and unit queue are bit-identical with mid-step samples (40 and 500 Hz) and noise; (4, 16) puts environments
    in the large tier"""
    n = 48
    res = []
    for mode in (0, 1, 2):
        env = make_env("Stack", n, mode, 9, **({"tier_small": tier} if tier else {}))
        _configure(env)
        env.modify_observable("robot0_joint_vel", "sampling_rate", 500)
        env.reset()
        acts = random_actions(env, 6)
        res.append(_masked_run(env, acts, 3) + tuple(env.sim.array(a).clone() for a in ("obs_timer", "obs_sampled", "obs_nsample")))
        env.close()
    for r in res[1:]:
        for a, b in zip(res[0], r):
            assert torch.equal(a, b)


def test_snapshots_carry_the_timers():
    n = 16
    env = make_env("Lift", n, 1, 2)
    _configure(env)
    env.reset()
    acts = random_actions(env, 6)
    run(env, acts[:3])
    state = env.get_env_state()
    assert {"obs_timer", "obs_sampled", "obs_nsample"} <= set(state["sim"].names)
    a = run(env, acts[3:]) + (env.sim.obs_nsample.clone(), env.sim.obs_timer.clone())
    env.set_env_state(state)
    b = run(env, acts[3:]) + (env.sim.obs_nsample.clone(), env.sim.obs_timer.clone())
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    # a clone takes the source's timers, flags and counts
    src = torch.arange(n, device=env.device).flip(0).to(torch.int32)
    before = {name: env.sim.array(name).clone() for name in ("obs_timer", "obs_sampled", "obs_nsample")}
    env.clone_envs(src)
    torch.cuda.synchronize()
    for name, t in before.items():
        assert torch.equal(env.sim.array(name), t[src.long()])
    plain = make_env("Lift", n, 1, 2)
    with pytest.raises(ValueError, match="signature"):
        plain.set_env_state(state)
    plain.close()
    env.close()


def test_masked_reset_restarts_the_timers_and_keeps_the_counts():
    n = 8
    env = make_env("Lift", n, 1, 5)
    _configure(env)
    env.reset()
    run(env, random_actions(env, 3))
    t0, s0, c0, obs0 = (env.sim.array(a).clone() for a in ("obs_timer", "obs_sampled", "obs_nsample", "obs"))
    mask = torch.zeros(n, dtype=torch.bool, device=env.device)
    mask[2] = mask[5] = True
    env.reset(mask=mask)
    torch.cuda.synchronize()
    t1, s1, c1, obs1 = (env.sim.array(a).clone() for a in ("obs_timer", "obs_sampled", "obs_nsample", "obs"))
    keep = ~mask
    assert torch.equal(t1[keep], t0[keep]) and torch.equal(s1[keep], s0[keep]) and torch.equal(c1[keep], c0[keep])
    assert torch.equal(obs1[keep], obs0[keep])
    assert torch.equal(c1[mask], c0[mask] + 1)  # the forced sample of every observable
    dt = env.model.opt_timestep
    periods = torch.tensor([1.0 / RATES[k % len(RATES)] for k in range(len(env._obs_slices))], dtype=torch.float64, device=env.device)
    expect = torch.where(periods <= dt, torch.fmod(torch.full_like(periods, dt), periods), torch.full_like(periods, dt))
    assert torch.equal(t1[mask], expect.expand(2, -1))
    env.close()


def test_library_argument_checks():
    from robosuite_b200.engine import B2SError, BatchedSim
    from tests.util import load

    sim = BatchedSim(load("Lift_Panda"), 2, precision="f32")
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
            sim.obs_modifiers([0, 0] + [0] * 31, mods)
    with pytest.raises(B2SError, match="out of range"):
        sim.obs_modifiers([0, 1], [ok])
    with pytest.raises(B2SError, match="out of range"):
        sim.obs_modifiers([0, -1], [ok, ok])
    sim.obs_modifiers([0, 1], [ok, (0.1, CORRUPT_NONE, 0, 0, 0, 0)], seed=3)
    assert sim.obs_timer.shape == (2, 2) and sim.obs_nsample.shape == (2, 2)
    assert {"obs_timer", "obs_sampled", "obs_nsample"} <= {s[0] for s in sim.snapshot_layout()[2]}
    sim.obs_modifiers([], [])
    assert not any(s[0] == "obs_timer" for s in sim.snapshot_layout()[2])
    sim.close()
