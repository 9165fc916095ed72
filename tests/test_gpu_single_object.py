"""GPU: the single-object PickPlace / NutAssembly variants and the per-environment object selection (b2s_obs_objects, OB_SEL_*):
lockstep with the CPU stand-in, the three schedules, snapshots, auto-reset and the ABI's errors."""
import numpy as np
import pytest

from tests.oracle_sim_select import SelectOracleSim
from tests.schedules import make_env, random_actions, run, switches
from tests.util import load

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

TASKS = ["PickPlaceMilk", "PickPlaceBread", "PickPlaceCereal", "PickPlaceCan", "PickPlaceSingle", "NutAssemblySingle"]


def _mirror_reset(cpu, dev, mask=None):
    """the CPU stand-in resets the masked environments into the device's sampled state and mode-1 draw"""
    q = dev._reset_qpos.detach().cpu().to(torch.float64)
    draw = getattr(dev, "_sel_draw", None)

    def sample(n):
        if draw is not None:
            cpu._sel_draw = draw.cpu()
        return q.clone()

    cpu._sample_reset_state = sample
    try:
        cpu.reset(None if mask is None else mask.cpu())
    finally:
        del cpu._sample_reset_state


@pytest.mark.parametrize("precision", ["f64", "f32"])
@pytest.mark.parametrize("task", TASKS)
def test_lockstep_with_the_cpu_stand_in(task, precision):
    """observations, rewards and qpos against the oracle-backed stand-in (gates of test_gpu_env.py's other-task test), with a masked
    reset after the second step that redraws the mode-1 objects"""
    import robosuite_b200 as suite

    n = 3
    kw = dict(robots="Panda", num_envs=n, seed=11, horizon=50, reward_shaping=True)
    dev = suite.make(task, precision=precision, **kw)
    cpu = suite.make(task, sim_cls=SelectOracleSim, precision="f64", **kw)
    _mirror_reset(cpu, dev)
    single = dev.single_object_mode == 1
    if single:
        assert torch.equal(cpu.object_id, dev.object_id.cpu())

    def compare(tag, rd=None, rc=None):
        a = dev._modality_slices["object-state"][0]  # the object rows, as test_gpu_env.py compares them
        od, oc = dev.sim.obs[:, a:].cpu().double().numpy(), cpu.sim.obs[:, a:].numpy()
        tol = 3e-3 if task.startswith("PickPlace") else 1e-3
        assert np.abs(od - oc).max() < tol, (task, tag, int(np.abs(od - oc).argmax()), float(np.abs(od - oc).max()))
        if rd is not None:
            assert np.abs(rd.cpu().double().numpy() - rc.numpy()).max() < 2e-3, (task, tag, rd, rc)
        qd, qc = dev.sim.qpos.cpu().double().numpy(), cpu.sim.qpos.numpy()
        assert max(np.abs(qd[e] - qc[e]).max() / np.abs(qc[e]).max() for e in range(n)) < 2e-3, (task, tag)

    compare("reset")
    rng = np.random.default_rng(1)
    mask = torch.tensor([True, False, True], device=dev.device)
    for t in range(4):
        act = rng.uniform(-1, 1, size=(n, 7))
        _, rd, _, _ = dev.step(torch.as_tensor(act))
        _, rc, _, _ = cpu.step(torch.as_tensor(act))
        compare(t, rd, rc)
        if t == 1:
            sel0 = dev.object_id.clone() if single else None
            dev.reset(mask)
            _mirror_reset(cpu, dev, mask)
            compare("masked reset")
            if single:
                assert torch.equal(dev.object_id[~mask], sel0[~mask])
                assert torch.equal(dev.object_id[mask], dev._sel_draw.to(torch.int32)[mask])
                assert torch.equal(cpu.object_id, dev.object_id.cpu())
    assert int(dev.sim.warn.abs().max()) == 0
    dev.close()


@pytest.mark.parametrize("task", ["PickPlaceSingle", "NutAssemblySingle"])
def test_schedules_agree_bit_for_bit(task):
    """fused kernel, pipeline and unit queue with a small tier of (4, 24): environments run in both tiers; a masked reset mid-run
    redraws objects.  The whole run stays inside switches(...): the pipeline reads B2S_NO_GJK_CACHE at its first step, and the GJK warm
    start (which the fused kernel does not have) moves mesh-object trajectories in the last bits"""
    res = []
    for mode in (0, 1, 2):
        with switches(gjk_cache=False, ctrl_split=False):
            env = make_env(task, 24, mode, 5, gjk_cache=False, ctrl_split=False, tier_small=(4, 24), reward_shaping=True)
            acts = random_actions(env, 6)
            r = run(env, acts[:3])
            mask = torch.zeros(env.num_envs, dtype=torch.bool, device=env.device)
            mask[::3] = True
            env.reset(mask=mask)
            res.append(r + (env.object_id.clone(),) + run(env, acts[3:]) + (env.sim.warn.clone(),))
            env.close()
    for r in res[1:]:
        for a, b in zip(res[0], r):
            assert torch.equal(a, b)


def test_snapshots_carry_the_selection():
    env = make_env("PickPlaceSingle", 8, 1, 3, horizon=10 ** 6, reward_shaping=True)
    names = env.sim.snapshot().names
    assert "obj_sel" in names
    acts = random_actions(env, 8)
    run(env, acts[:2])
    st = env.get_env_state()
    sel = env.object_id.clone()
    ref = run(env, acts[2:])
    ref_sel = env.object_id.clone()
    # scramble the selection, then restore
    env.sim.obj_sel.copy_((sel + 1) % 4)
    env.set_env_state(st)
    assert torch.equal(env.object_id, sel)
    got = run(env, acts[2:])
    for a, b in zip(ref, got):
        assert torch.equal(a, b)
    assert torch.equal(env.object_id, ref_sel)
    # clones take their source's object and continue as the source does
    env.set_env_state(st)
    src = [5, 5, 5, 5, -1, -1, -1, -1]
    env.clone_envs(src)
    take = torch.as_tensor([5, 5, 5, 5, 4, 5, 6, 7], device=env.device)
    assert torch.equal(env.object_id, sel[take])
    got = run(env, acts[2:, take])
    for a, b in zip(ref, got):
        assert torch.equal(a[take], b)
    env.close()


def test_handles_without_a_list_keep_their_snapshot_layout():
    env = make_env("PickPlace", 4, 1, 3)
    names = env.sim.snapshot().names
    assert "obj_sel" not in names
    env.close()


def test_gym_wrapper_auto_reset_redraws_exactly_the_finished_environments():
    from robosuite_b200.wrappers import BatchedGymWrapper

    env = make_env("PickPlaceSingle", 8, 1, 7, horizon=10 ** 6)
    env.horizon = 4
    g = BatchedGymWrapper(env)
    g.reset()
    env.set_episode_steps(np.array([0, 2, 0, 2, 0, 2, 0, 2]))
    redrawn = 0
    for t in range(4):
        before = env.object_id.clone()
        env._sel_draw = None
        _, _, term, trunc, _ = g.step(torch.zeros((8, 7), device=env.device))
        done = (torch.as_tensor(term) | torch.as_tensor(trunc)).to(env.device).bool()
        assert torch.equal(env.object_id[~done], before[~done])
        if bool(done.any()):
            assert env._sel_draw is not None
            assert torch.equal(env.object_id[done], env._sel_draw.to(torch.int32)[done])
            redrawn += int(done.sum())
    assert redrawn == 8  # every environment finished once: the odd ones at the second step, the even ones at the fourth
    g.close()


def test_abi_errors_and_out_of_range_selection():
    from robosuite_b200 import controller_config as cc
    from robosuite_b200.engine import B2SError, BatchedSim, CtrlCfg
    from robosuite_b200.envs.base import OB_BODY_POS, OB_QPOS, OB_SEL_BODY_POS, OB_SEL_INDEX

    model = load("PickPlace_Panda")
    bn, jn = model.names["body"], model.names["joint"]
    free = [bn.index(n + "_main") for n in ("Milk", "Bread", "Cereal", "Can")]
    hand = bn.index("robot0_right_hand")
    n = 6
    sim = BatchedSim(model, n, precision="f64")
    sim.ctrl_config(cc.resolve(model, cc.default_composite_config(), CtrlCfg))
    sel_ops = ([OB_SEL_BODY_POS] * 3 + [OB_SEL_INDEX], [0] * 4, [0, 1, 2, 0])
    with pytest.raises(B2SError):  # a selection op without a list
        sim.obs_config(*sel_ops)
    for bad in ([hand], [0], [len(bn)], [-1], free + [free[0]]):  # no free joint, the world, out of range, n > 4
        with pytest.raises(B2SError):
            sim.obs_objects(bad)
    sel = sim.obs_objects(free)
    assert sel.dtype == torch.int32 and sel.shape == (n,) and int(sel.abs().max()) == 0
    sim.obs_config(*sel_ops)
    with pytest.raises(B2SError):  # clearing a list the table reads
        sim.obs_objects([])
    sel.copy_(torch.tensor([0, 1, 2, 3, 9, -1], dtype=torch.int32))
    q = sim.qpos.clone()
    sim.reset_envs(None, q)
    torch.cuda.synchronize()
    obs, warn, xpos = sim.obs.cpu().numpy(), sim.warn.cpu().numpy(), sim.xpos.cpu().numpy()
    for e in range(4):
        assert np.array_equal(obs[e, :3], xpos[e, free[e]]) and obs[e, 3] == e and not warn[e] & 512
    for e in (4, 5):  # (objects stacked at qpos0 may raise other bits too)
        assert np.array_equal(obs[e], np.zeros(4)) and warn[e] & 512
    # a handle whose tables do not use the selection may clear its list; one whose task table reads it may not
    sim2 = BatchedSim(model, 2, precision="f32")
    with pytest.raises(B2SError):  # a task table with a selection op and no list
        sim2.task_table([(OB_SEL_BODY_POS, 0, 0)])
    sim2.obs_objects(free[:2])
    sim2.obs_config([OB_QPOS, OB_BODY_POS], [0, free[0]], [0, 0])
    sim2.task_table([(OB_SEL_BODY_POS, 0, 0), (OB_SEL_INDEX, 0, 0)])
    with pytest.raises(B2SError):  # clearing a list the task table reads
        sim2.obs_objects([])
    sim2.task_table([(OB_BODY_POS, free[1], 0)])
    assert sim2.obs_objects([]) is None
    sim.close()
    sim2.close()
