"""Object placement on the device (b2s_place_config / b2s_place_objects, make(..., placement_initializer=...)): the q rows and
the Door's pose overrides against the numpy restatement (tests/placement_ref.py) bit for bit, independence of the batch size and
the mask, masked resets, the distributions and the overlap rule at 4096 environments, warn bit 1024, every task against the oracle
from the restated placements, and the auto-resetting gym wrapper without a device read."""
import math

import numpy as np
import pytest

torch = pytest.importorskip("torch")

from robosuite_b200.placement_samplers import SequentialCompositeSampler, UniformRandomSampler, lower  # noqa: E402
from tests.placement_ref import place_values  # noqa: E402
from tests.util import load  # noqa: E402

pytestmark = pytest.mark.gpu

SEED, N = 0x1234_5678_9ABC_DEF0, 37


def _free_objects(model, k):
    """k of the model's free joints as placement objects with made-up box metadata"""
    adr = [int(model.jnt_qposadr[j]) for j in range(len(model.jnt_type)) if int(model.jnt_type[j]) == 0][:k]
    meta = [(0.03, -0.02, 0.02), (0.04, -0.025, 0.025), (0.05, -0.05, 0.05), (0.02, -0.01, 0.03)]
    return {"o%d" % i: dict(radius=meta[i][0], bottom=meta[i][1], top=meta[i][2], qpos_adr=a, body=-1) for i, a in enumerate(adr)}


def _samplers():
    """every option: inverted ranges, boundary shrink, validity on / off, each rotation form, each axis, reference by name with and
    without on_top, a vector reference, composites and hide; the last one is nearly impossible (thousands of tries)"""
    out = [UniformRandomSampler("U", mujoco_objects=["o0", "o1", "o2"], x_range=(-0.1, 0.1), y_range=(0.1, -0.1),
                                reference_pos=(0.0, 0.0, 0.8), z_offset=0.01),
           UniformRandomSampler("X", mujoco_objects=["o0", "o1", "o2"], x_range=(-0.08, 0.08), y_range=(-0.08, 0.08), rotation=(0.2, -0.4),
                                rotation_axis="x", ensure_object_boundary_in_range=False, ensure_valid_placement=False)]
    c = SequentialCompositeSampler("C")
    c.append_sampler(UniformRandomSampler("A", mujoco_objects="o0", x_range=(-0.02, 0.02), y_range=(-0.02, 0.02),
                                          rotation=[(0, 0.5), (2, 3), (-1, -0.5)], rotation_axis="y", reference_pos=(0.1, -0.1, 0.8)))
    c.append_sampler(UniformRandomSampler("B", mujoco_objects="o1", rotation=1.25, ensure_object_boundary_in_range=False),
                     sample_args={"reference": "o0"})
    c.append_sampler(UniformRandomSampler("B2", mujoco_objects="o3", x_range=(-0.01, 0.01)), sample_args={"reference": "o1", "on_top": False})
    c.hide("o2")
    out.append(c)
    d = SequentialCompositeSampler("D")
    d.append_sampler(UniformRandomSampler("A", mujoco_objects=["o0", "o1", "o2"], x_range=(-0.062, 0.062), y_range=(-0.062, 0.062),
                                          ensure_object_boundary_in_range=False), sample_args={"reference": (0.0, 0.0, 0.8)})
    out.append(d)
    return out


def _masks(n, dev):
    r = np.random.default_rng(3)
    return [None, torch.as_tensor(np.arange(n) % 3 == 1), torch.as_tensor(r.random(n) < 0.5)]


@pytest.mark.parametrize("k", range(4))
def test_q_rows_equal_the_restatement_bit_for_bit(k):
    from robosuite_b200.engine import BatchedSim

    model = load("PickPlace_Panda")
    sampler = _samplers()[k]
    objs = _free_objects(model, 4)
    objs = {n: objs[n] for n in sampler.mujoco_objects}
    _, entries = lower(sampler, objs)
    rows = {}
    for prec in ("f64", "f32"):
        sim = BatchedSim(model, N, precision=prec)
        sim.place_config(entries)
        q = torch.full((N, model.nq), -7.0, dtype=torch.float64, device="cuda")
        qh = q.cpu().numpy()
        for c, mask in enumerate(_masks(N, sim.torch_device)):
            m8 = None if mask is None else mask.to(device="cuda", dtype=torch.uint8)
            sim.place_objects(q, m8, SEED, c)
            envs = range(N) if mask is None else np.nonzero(mask.numpy())[0]
            place_values(entries, envs, SEED, c, qpos=qh)
            assert np.array_equal(q.cpu().numpy(), qh), (prec, c)  # masked rows placed, the others untouched
        rows[prec] = q.cpu()
        sim.close()
    assert torch.equal(rows["f64"], rows["f32"])


@pytest.mark.parametrize("prec", ["f64", "f32"])
def test_door_overrides_equal_the_restatement(prec):
    from robosuite_b200.engine import BatchedSim

    model = load("Door_Panda")
    bn = model.names["body"]
    main, frame = bn.index("Door_main"), bn.index("Door_frame")
    s = UniformRandomSampler("S", mujoco_objects="Door", x_range=(0.05, 0.1), y_range=(-0.02, 0.02), rotation=[(-1.8, -1.3), (0.2, 0.3)],
                             ensure_object_boundary_in_range=False, reference_pos=(-0.2, -0.35, 0.8))
    _, entries = lower(s, {"Door": dict(radius=0.3, bottom=-0.3, top=0.3, qpos_adr=-1, body=main)})
    sim = BatchedSim(model, N, precision=prec)
    (pm, qm), (pf, qf) = sim.body_pose_override(main), sim.body_pose_override(frame)
    sim.place_config(entries)
    local = [(np.asarray(model.body_pos[frame], dtype=np.float64), np.asarray(model.body_quat[frame], dtype=np.float64))]
    dt = np.float64 if prec == "f64" else np.float32
    want = [t.cpu().numpy().copy() for t in (pm, qm, pf, qf)]
    for c, mask in enumerate(_masks(N, sim.torch_device)):
        sim.place_objects(None, None if mask is None else mask.to(device="cuda", dtype=torch.uint8), SEED, c)
        envs = list(range(N)) if mask is None else list(np.nonzero(mask.numpy())[0])
        res = place_values(entries, envs, SEED, c, ov_local={0: local})
        for i, e in enumerate(envs):
            (p0, q0), (p1, q1) = res["ov"][0][i]
            for arr, v in zip(want, (p0, q0, p1, q1)):
                arr[e] = np.asarray(v, dtype=np.float64).astype(dt)  # rounded to the handle's precision last
        for t, w in zip((pm, qm, pf, qf), want):
            assert np.array_equal(t.cpu().numpy(), w), (prec, c)
    sim.close()


def test_placements_do_not_depend_on_the_batch_size():
    from robosuite_b200.engine import BatchedSim

    model = load("PickPlace_Panda")
    sampler = _samplers()[0]
    _, entries = lower(sampler, {n: v for n, v in _free_objects(model, 3).items()})
    out = []
    for n in (5, 4096):
        sim = BatchedSim(model, n, precision="f32")
        sim.place_config(entries)
        q = torch.zeros((n, model.nq), dtype=torch.float64, device="cuda")
        sim.place_objects(q, None, SEED, 9)
        out.append(q[:5].cpu())
        sim.close()
    assert torch.equal(out[0], out[1])


def _make(task, n, sampler, **kw):
    import robosuite_b200 as suite

    return suite.make(task, robots="Panda", num_envs=n, seed=11, placement_initializer=sampler, **kw)


def _stack_sampler():
    return UniformRandomSampler("S", x_range=(-0.12, 0.12), y_range=(-0.1, 0.1), rotation=(-0.5, 0.5), reference_pos=(0, 0, 0.8),
                                z_offset=0.01)


def test_masked_reset_leaves_the_other_environments_bit_identical():
    n = 64
    a, b = _make("Stack", n, _stack_sampler()), _make("Stack", n, _stack_sampler())
    gen = torch.Generator(device=a.device)
    gen.manual_seed(0)
    acts = torch.rand((10, n, a.action_dim), generator=gen, device=a.device, dtype=a.dtype) * 2 - 1
    for t in range(4):
        a.step(acts[t])
        b.step(acts[t])
    mask = torch.zeros(n, dtype=torch.bool, device=a.device)
    mask[2::5] = True
    before = {k: getattr(a.sim, k).clone() for k in ("qpos", "qvel", "obs", "ctrl_goal_pos")}
    a.reset(mask=mask)
    for k, v in before.items():
        assert torch.equal(v[~mask], getattr(a.sim, k)[~mask]), k
    names, entries = lower(a.placement_initializer, a._placement_objects())
    qh = np.zeros((n, a.model.nq))
    place_values(entries, np.nonzero(mask.cpu().numpy())[0], a._place_seed, 1, qpos=qh)
    for e in entries:
        adr = e["qpos_adr"]
        got = a._reset_qpos[mask][:, adr:adr + 7].double().cpu().numpy()
        assert np.array_equal(got, qh[mask.cpu().numpy()][:, adr:adr + 7].astype(np.float32).astype(np.float64))
    for t in range(4, 10):
        a.step(acts[t])
        b.step(acts[t])
    assert torch.equal(a.sim.qpos[~mask], b.sim.qpos[~mask]) and torch.equal(a.sim.obs[~mask], b.sim.obs[~mask])
    assert int(a.sim.warn.abs().max()) == 0


def test_distributions_and_overlap_rule_at_4096_environments():
    from scipy import stats

    n = 4096
    env = _make("Stack", n, _stack_sampler())
    q = env._reset_qpos.double().cpu().numpy()
    A, B = env.cubeA_qadr, env.cubeB_qadr
    rA = float(np.linalg.norm(env.half["A"][:2]))
    lo, hi = -0.12 + rA, 0.12 - rA
    assert stats.kstest((q[:, A] - lo) / (hi - lo), "uniform").pvalue > 1e-3
    lo, hi = -0.1 + rA, 0.1 - rA
    assert stats.kstest((q[:, A + 1] - lo) / (hi - lo), "uniform").pvalue > 1e-3
    yaw = 2 * np.arctan2(q[:, A + 6], q[:, A + 3])
    assert stats.kstest((yaw + 0.5) / 1.0, "uniform").pvalue > 1e-3
    rB = float(np.linalg.norm(env.half["B"][:2]))
    d = np.hypot(q[:, A] - q[:, B], q[:, A + 1] - q[:, B + 1])
    assert (d > (rA + rB) * (1 - 1e-6)).all()  # f32 rows: the rule holds in fp64 before rounding
    assert int(env.sim.warn.abs().max()) == 0


def test_impossible_sampler_sets_warn_bit_1024_without_a_fault():
    s = UniformRandomSampler("S", x_range=(0, 0.001), y_range=(0, 0.001), ensure_object_boundary_in_range=False, reference_pos=(0, 0, 0.8))
    env = _make("Stack", 256, s)
    torch.cuda.synchronize()
    assert (env.sim.warn == 1024).all()
    feasible = _stack_sampler()
    feasible.add_objects(["cubeA", "cubeB"])
    names, entries = lower(feasible, env._placement_objects())
    env.sim.place_config(entries)  # a feasible program in the same handle
    env.reset()
    assert int(env.sim.warn.abs().max()) == 0


def _sampler_for(task):
    if task == "Door":
        return UniformRandomSampler("S", x_range=(0.05, 0.1), y_range=(-0.03, 0.03), rotation=(-math.pi / 2 - 0.3, -math.pi / 2 + 0.1),
                                    ensure_object_boundary_in_range=False, reference_pos=(-0.2, -0.35, 0.8))
    if task.startswith("Nut"):
        c = SequentialCompositeSampler("N")
        c.append_sampler(UniformRandomSampler("Sq", mujoco_objects="SquareNut", x_range=(-0.14, -0.1), y_range=(0.1, 0.24),
                                              ensure_object_boundary_in_range=False, reference_pos=(0, 0, 0.82), z_offset=0.02))
        c.append_sampler(UniformRandomSampler("Ro", mujoco_objects="RoundNut", x_range=(-0.14, -0.1), y_range=(-0.24, -0.1),
                                              ensure_object_boundary_in_range=False, reference_pos=(0, 0, 0.82), z_offset=0.02))
        return c
    return _stack_sampler()


@pytest.mark.parametrize("task", ["Lift", "Stack", "NutAssemblyRound", "NutAssemblySquare", "NutAssemblySingle", "Door"])
def test_tasks_reset_to_the_restated_placements_and_follow_the_oracle(task):
    from tests.oracle_sim_placement import PlacementOracleSim

    n = 4
    env = _make(task, n, _sampler_for(task), precision="f64")
    names, entries = lower(env.placement_initializer, env._placement_objects())
    q = env._reset_qpos.cpu().numpy()
    if task == "Door":
        res = place_values(entries, range(n), env._place_seed, 0, ov_local={0: [env._frame_local]})
        for e in range(n):
            (p0, q0), _ = res["ov"][0][e]
            assert env.door_pose[0][e].tolist() == [float(v) for v in p0] and env.door_pose[1][e].tolist() == [float(v) for v in q0]
    else:
        qh = np.zeros_like(q)
        place_values(entries, range(n), env._place_seed, 0, qpos=qh)
        sel = env._sel_draw.cpu().numpy() if getattr(env, "single_object_mode", 0) == 1 else None
        for i, e in enumerate(entries):
            a = e["qpos_adr"]
            for k in range(n):
                parked = (sel is not None and sel[k] != i) or (getattr(env, "single_object_mode", 0) == 2 and i != env.nut_id)
                assert parked or np.array_equal(q[k, a:a + 7], qh[k, a:a + 7]), (task, i, k)
    o = _make(task, n, _sampler_for(task), precision="f64", sim_cls=PlacementOracleSim)
    if task == "Door":
        for dst, src in zip(o._door_ov, env._door_ov):
            for d, s_ in zip(dst, src):
                d.copy_(s_.cpu())
    if getattr(env, "_sel", None) is not None:
        o._sel.copy_(env._sel.cpu())
    o.reset_to(env._reset_qpos.cpu())
    env.reset_to(env._reset_qpos)
    gen = np.random.default_rng(2)
    for _ in range(3):
        act = gen.uniform(-1, 1, size=(n, env.action_dim))
        env.step(torch.as_tensor(act, device=env.device))
        o.step(torch.as_tensor(act))
    assert np.abs(env.sim.qpos.cpu().numpy() - o.sim.qpos.numpy()).max() < 1e-4


def test_gym_wrapper_autoreset_replaces_exactly_the_finished_environments():
    from robosuite_b200.wrappers import BatchedGymWrapper

    n, H = 32, 5
    env = _make("Lift", n, UniformRandomSampler("S", x_range=(-0.1, 0.1), y_range=(-0.1, 0.1), reference_pos=(0, 0, 0.8), z_offset=0.01),
                horizon=H)
    w = BatchedGymWrapper(env)
    w.reset()
    env.set_episode_steps(np.arange(n) % H)
    acts = torch.zeros((2 * H, n, env.action_dim), device=env.device, dtype=env.dtype)
    names, entries = lower(env.placement_initializer, env._placement_objects())
    a = env.cube_qadr
    torch.cuda.synchronize()
    records = []
    with torch.cuda.stream(torch.cuda.current_stream()):
        torch.cuda.set_sync_debug_mode("error")
        try:
            for t in range(2 * H):
                c0 = env._place_counter
                w.step(acts[t])
                records.append((c0, env._place_counter, env._reset_qpos.clone()))
        finally:
            torch.cuda.set_sync_debug_mode("default")
    steps = np.arange(n) % H
    for c0, c1, rq in records:
        steps = steps + 1
        done = steps >= H
        assert c1 == c0 + int(done.any())
        if done.any():
            qh = np.zeros((n, env.model.nq))
            place_values(entries, np.nonzero(done)[0], env._place_seed, c0, qpos=qh)
            got = rq[torch.as_tensor(done, device=rq.device)][:, a:a + 7].double().cpu().numpy()
            assert np.array_equal(got, qh[done][:, a:a + 7].astype(np.float32).astype(np.float64))
        steps[done] = 0
    assert int(env.sim.warn.abs().max()) == 0
