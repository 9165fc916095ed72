"""Whole-environment snapshots (b2s_snapshot / b2s_restore, BatchedSim.snapshot / restore / clone_envs, the environment layer's
get_env_state / set_env_state / clone_envs): a restored environment continues bit-identically to its source under the same actions,
whatever the batch around it.  The rollouts are contact-rich scripted Lift rollouts (tests/schedules.py, lift_actions: random arm
actions, gripper closing, half of the arms pushing down onto the table / cube), fp32 with the GJK warm start on unless noted."""
import numpy as np
import pytest

from tests.schedules import lift_actions, make_env

pytestmark = pytest.mark.gpu


def _run(env, acts):
    import torch

    out = []
    for a in acts:
        _, r, d, _ = env.step(torch.as_tensor(a, dtype=env.dtype, device=env.device))
        out.append((r.clone(), d.clone()))
    return out


def _rows(env):
    import torch

    torch.cuda.synchronize()
    return env.sim.snapshot().rows.cpu().numpy()


def _differing(env, a, b):
    """names of the sections in which two snapshot rows differ"""
    from robosuite_b200.engine import _ITEMSIZE

    return [n for n, off, cnt, dt in env.sim.snapshot_layout()[2]
            if not np.array_equal(a[..., off:off + cnt * _ITEMSIZE[dt]], b[..., off:off + cnt * _ITEMSIZE[dt]])]


def _warm(env, steps=10, seed=5):
    _run(env, lift_actions(steps, env.num_envs, seed=seed, dim=env.action_dim))


# the task draws the cube's mass and moments itself (per_env_cube_size); the wrapper randomises everything else
_TASK_DRAWS_CUBE = {"randomize_mass": False, "randomize_inertia": False}

LIVE = ("qpos", "qvel", "qacc", "qacc_warmstart", "obs", "task_out", "ctrl", "ctrl_goal_pos", "ctrl_goal_ori", "ctrl_initial_joint",
        "ctrl_grip_state", "ctrl_jv_state", "ctrl_torque", "warn")


@pytest.mark.parametrize("mode, precision", [(0, "f32"), (1, "f32"), (2, "f32"), (1, "f64")],
                         ids=["fused", "pipeline", "unit_queue", "pipeline_f64"])
def test_round_trip_bit_exact(mode, precision):
    """snapshot, 20 control steps, restore, the same 20 steps again: every state array, the observation and task rows, the controller
    state, the warn bits and the whole snapshot row (GJK cache included) are bit-identical to the first run"""
    env = make_env("Lift", 16, mode, 11, horizon=10 ** 6, precision=precision)
    _warm(env)
    acts = lift_actions(20, env.num_envs)
    snap = env.sim.snapshot()
    _run(env, acts)
    first = {k: env.sim.array(k).cpu().numpy().copy() for k in LIVE}
    rows1 = _rows(env)
    env.sim.restore(snap)
    _run(env, acts)
    for k in LIVE:
        assert np.array_equal(env.sim.array(k).cpu().numpy(), first[k]), k
    rows2 = _rows(env)
    assert np.array_equal(rows2, rows1), _differing(env, rows2, rows1)
    assert np.isfinite(first["qpos"]).all() and int(np.abs(first["warn"]).max()) == 0
    env.close()


def _clone_checks(env, steps=20):
    """from one saved batch state S: a plain run (per-environment actions), then runs from S with clones; every cloned environment
    ends with exactly its source's row of the plain run"""
    n = env.num_envs
    acts = lift_actions(steps, n, dim=env.action_dim)
    S = env.sim.snapshot()
    _run(env, acts)
    base = _rows(env)
    assert int(np.abs(env.sim.warn.cpu().numpy()).max()) == 0
    cases = {"env 3 everywhere": np.full(n, 3), "reversed": np.arange(n)[::-1].copy(),
             "half kept": np.where(np.arange(n) < n // 2, -1, 3)}
    for what, src in cases.items():
        env.sim.restore(S)
        env.clone_envs(src)
        take = np.where(src < 0, np.arange(n), src)
        _run(env, acts[:, take])
        got = _rows(env)
        assert np.array_equal(got, base[take]), (what, _differing(env, got, base[take]))
        if what == "env 3 everywhere":
            assert (got == got[:1]).all()
    return S


def test_clone_bit_exact():
    """env 3 cloned into all 16 environments stays identical to itself and to env 3's own run; a reversed permutation gives the
    reversed trajectories; environments with src = -1 are bit-identical to a run without any restore"""
    env = make_env("Lift", 16, 1, 11, horizon=10 ** 6)
    _warm(env)
    _clone_checks(env)
    env.close()


@pytest.mark.parametrize("mode", [1, 2], ids=["pipeline", "unit_queue"])
def test_cross_handle_bit_exact(mode):
    """env 5 of a 16-environment handle, restored into a 1-environment handle and into every environment of a 13-environment handle
    with 8 groups and no small tail tier, continues bit-identically for 40 control steps"""
    import torch

    src = make_env("Lift", 16, mode, 11, horizon=10 ** 6)
    _warm(src)
    snap = src.sim.snapshot([5])
    acts = lift_actions(40, 16)
    one = make_env("Lift", 1, mode, 11, horizon=10 ** 6)
    many = make_env("Lift", 13, mode, 11, groups=8, horizon=10 ** 6, tier_small=(48, 128))
    one.sim.restore(snap, torch.zeros(1, dtype=torch.int32, device=one.device))
    many.sim.restore(snap, np.zeros(13, dtype=np.int32))
    for t in range(40):
        _run(src, acts[t:t + 1])
        _run(one, acts[t:t + 1, 5:6])
        _run(many, np.repeat(acts[t:t + 1, 5:6], 13, axis=1))
        if t % 10 == 9:
            ref = _rows(src)[5]
            got1, got13 = _rows(one), _rows(many)
            assert np.array_equal(got1[0], ref), (t, _differing(src, got1[0], ref))
            assert (got13 == ref).all(), (t, _differing(src, got13, ref[None].repeat(13, 0)))
    for e in (src, one, many):
        e.close()


def test_overrides_are_carried():
    """Lift with per-environment cubes under dynamics randomisation: clones carry sizes, masses, moments, friction, solref / solimp,
    the dof vectors and the derived constants, and continue bit-identically"""
    import torch

    from robosuite_b200.wrappers import BatchedDomainRandomizationWrapper

    w = BatchedDomainRandomizationWrapper(make_env("Lift", 16, 1, 4, horizon=10 ** 6, per_env_cube_size=True),
                                          seed=2, randomize_every_n_steps=0, dynamics_randomization_args=_TASK_DRAWS_CUBE)
    w.reset()
    env = w.env
    _warm(env)
    names = [n for n, *_ in env.sim.snapshot_layout()[2]]
    for f in ("geom_size:", "geom_friction:", "geom_solref:", "geom_solimp:", "body_mass:", "body_inertia:"):
        assert any(n.startswith(f) for n in names), f
    for f in ("dof_damping", "dof_armature", "dof_frictionloss", "dof_invweight0", "body_invweight0", "meaninertia"):
        assert f in names, f
    S = _clone_checks(env)
    env.sim.restore(S)
    before = env.sim.snapshot()
    env.clone_envs(np.full(16, 7))
    after = env.sim.snapshot()
    torch.cuda.synchronize()
    differed = set()
    for n in names:
        a, b = after.field(n), before.field(n)
        assert torch.equal(a, b[7:8].expand_as(b)), n
        if not torch.equal(b, b[7:8].expand_as(b)):
            differed.add(n.split(":")[0])
    # the environments really differed before the clone
    assert {"geom_size", "geom_friction", "geom_solref", "body_mass", "body_inertia", "dof_damping", "dof_invweight0"} <= differed
    w.close()


def test_door_pose_overrides_are_carried():
    import torch

    env = make_env("Door", 8, 1, 11, horizon=10 ** 6)
    _warm(env)
    names = [n for n, *_ in env.sim.snapshot_layout()[2]]
    assert any(n.startswith("body_xpos_ov:") for n in names) and any(n.startswith("body_xquat_ov:") for n in names)
    pos = env.door_pose[0]
    assert not torch.equal(pos, pos[2:3].expand_as(pos))
    _clone_checks(env, steps=12)
    env.clone_envs(np.full(8, 2))
    for a in env.door_pose:
        assert torch.equal(a, a[2:3].expand_as(a))
    env.close()


def test_pick_place_env_state_clone():
    """PickPlace: clones reproduce their source's rewards, `done`, episode clock and objects_in_bins step by step"""
    import torch

    env = make_env("PickPlace", 8, 1, 11, horizon=10 ** 6, reward_shaping=True)
    env.horizon = 22  # the 10 warm-up steps and 12 more reach it
    _warm(env)
    acts = lift_actions(12, 8)
    st = env.get_env_state()
    ref = _run(env, acts)
    ref_bins = env.objects_in_bins.clone()
    ref_t = env.timestep.clone()
    env.set_env_state(st)
    env.clone_envs([6, 6, 6, 6, -1, -1, -1, -1])
    take = np.array([6, 6, 6, 6, 4, 5, 6, 7])
    got = _run(env, acts[:, take])
    idx = torch.as_tensor(take, device=env.device)
    for (r0, d0), (r1, d1) in zip(ref, got):
        assert torch.equal(r1, r0[idx]) and torch.equal(d1, d0[idx])
    assert bool(got[-1][1].all())  # the clocks reached the horizon on the source's schedule
    assert torch.equal(env.timestep, ref_t[idx]) and torch.equal(env.objects_in_bins, ref_bins[idx])
    env.close()


@pytest.mark.parametrize("device_src", [False, True], ids=["host_src", "device_src"])
def test_gym_wrapper_resets_clones_on_source_schedule(device_src):
    import torch

    from robosuite_b200.wrappers import BatchedGymWrapper

    env = make_env("Lift", 8, 1, 11, horizon=10 ** 6)
    env.horizon = 10
    g = BatchedGymWrapper(env)
    g.reset()
    env.set_episode_steps(np.arange(8))  # env e is e steps into its episode
    src = np.array([7, 7, 7, 7, -1, -1, -1, -1])
    g.clone_envs(torch.as_tensor(src, dtype=torch.int32, device=env.device) if device_src else src)
    assert (env._host_steps is None) == device_src
    clocks = []
    for t in range(6):
        _, _, term, _, info = g.step(torch.zeros((8, 7), device=env.device))
        clocks.append(env.timestep.cpu().numpy().copy())
        if t == 2:  # env 7 (and its clones) reached the horizon at their third step and were reset
            assert term.cpu().numpy().tolist() == [True] * 4 + [False] * 3 + [True] and "final_observation" in info
    clocks = np.array(clocks)
    assert (clocks[:, :4] == clocks[:, 7:8]).all()
    assert clocks[:, 7].tolist() == [8, 9, 0, 1, 2, 3] and clocks[:, 6].tolist() == [7, 8, 9, 0, 1, 2]
    g.close()


def test_signature_mismatch_raises():
    """another task, another precision, another override set, and an observation table configured after the snapshot"""
    from robosuite_b200.engine import BatchedSim
    from robosuite_b200.envs.lift import BatchedLift
    from tests.util import load

    a = make_env("Lift", 4, 1, 11, horizon=10 ** 6)
    snap = a.sim.snapshot()
    for other in (make_env("Stack", 4, 1, 11, horizon=10 ** 6), make_env("Lift", 4, 1, 11, horizon=10 ** 6, precision="f64"),
                  BatchedLift(robots="Panda", num_envs=4, seed=1, per_env_cube_size=True)):
        with pytest.raises(ValueError, match="signature"):
            other.sim.restore(snap)
        other.close()
    a.close()
    sim = BatchedSim(load("Lift_Panda"), 4)
    early = sim.snapshot()
    sim.obs_config([0, 0], [0, 1], [0, 0])
    with pytest.raises(ValueError, match="obs"):
        sim.restore(early)
    sim.close()


def test_bad_indices():
    """a host index out of range is an error; a device source row out of range (or below -1) leaves its environment bit-identical
    and sets warn bit 256 there only"""
    import torch

    from robosuite_b200.engine import B2SError

    env = make_env("Lift", 8, 1, 11, horizon=10 ** 6)
    _warm(env)
    with pytest.raises(B2SError):
        env.sim.snapshot([0, 8])
    two = env.sim.snapshot([0, 1])
    before = _rows(env)
    warn_off = [o for n, o, *_ in two.sections if n == "warn"][0]
    src = torch.full((8,), -1, dtype=torch.int32, device=env.device)
    src[4], src[6] = 2, -2
    env.sim.restore(two, src)
    after = _rows(env)
    w = env.sim.warn.cpu().numpy()
    assert w.tolist() == [0, 0, 0, 0, 256, 0, 256, 0]
    mask = np.ones(after.shape[1], dtype=bool)
    mask[warn_off:warn_off + 4] = False
    assert np.array_equal(after[:, mask], before[:, mask])
    env.close()


def test_field_decode_and_layout():
    """Snapshot.field(name) equals the live array of every section that has one; sections are 16-byte aligned, disjoint, in order
    and cover the row"""
    import torch

    from robosuite_b200.engine import B2SError, _ITEMSIZE
    from robosuite_b200.envs.lift import BatchedLift
    from robosuite_b200.wrappers import BatchedDomainRandomizationWrapper

    w = BatchedDomainRandomizationWrapper(BatchedLift(robots="Panda", num_envs=6, seed=3, per_env_cube_size=True), seed=1,
                                          randomize_every_n_steps=2, dynamics_randomization_args=_TASK_DRAWS_CUBE)
    w.reset()
    _run(w, lift_actions(5, 6))
    snap = w.env.sim.snapshot()
    torch.cuda.synchronize()
    checked = 0
    for name, *_ in snap.sections:
        try:
            live = w.env.sim.array(name)
        except B2SError:
            continue
        assert torch.equal(snap.field(name), live.reshape(6, -1)), name
        checked += 1
    assert checked >= len(snap.sections) - 6  # gjk_cache and the geom_size of slots declared through their friction only
    end = 0
    for name, off, cnt, dt in snap.sections:
        assert off % 16 == 0 and off == (end + 15) // 16 * 16, name
        end = off + cnt * _ITEMSIZE[dt]
    assert snap.rows.shape[1] == (end + 15) // 16 * 16
    w.close()
