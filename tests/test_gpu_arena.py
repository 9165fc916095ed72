"""Arena arguments on the device: tree pose overrides (b2s_body_pose_override_tree) and per-environment tables
(table_full_size / table_friction as [num_envs, 3], set_table) against batch-wide tables built from the same values."""
import ctypes as C

import numpy as np
import pytest

import robosuite_b200 as suite
from robosuite_b200.engine import B2SError, BatchedSim, lib
from robosuite_b200.mjcf.compiler import quat2mat, quat_mul
from tests.util import load

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

DEFAULT_SIZE, DEFAULT_FRICTION = (0.8, 0.8, 0.05), (1.0, 5e-3, 1e-4)


def _actions(env, steps, seed=4):
    g = np.random.default_rng(seed)
    return [torch.as_tensor(g.uniform(-1, 1, (env.num_envs, env.action_dim)), dtype=env.dtype, device=env.device) for _ in range(steps)]


def _rollout(env, steps, seed=4):
    out = []
    for a in _actions(env, steps, seed):
        obs, r, _, _ = env.step(a)
        out.append((env.flat_obs().clone(), r.clone(), env.sim.qpos.clone()))
    return out


def _make(n=8, mode=1, prec="f64", **kw):
    env = suite.make("Lift", robots="Panda", num_envs=n, seed=11, precision=prec, **kw)
    env.sim.set_mode(mode)
    env.reset()
    return env


@pytest.mark.parametrize("prec", ["f64", "f32"])
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_default_arguments_change_no_bit(mode, prec):
    a = _make(mode=mode, prec=prec)
    b = _make(mode=mode, prec=prec, table_full_size=DEFAULT_SIZE, table_friction=DEFAULT_FRICTION)
    for x, y in zip(_rollout(a, 20), _rollout(b, 20)):
        for u, v in zip(x, y):
            assert torch.equal(u, v)
    a.close()
    b.close()


def _welded_below(m, root):
    out = []
    for b in range(1, m.nbody):
        k = b
        while k > 0 and k != root:
            k = int(m.body_parentid[k])
        if k == root and b != root and int(m.body_weldid[b]) == 0:
            out.append(b)
    return out


def _rel_pose(m, root, b):
    chain, k = [], b
    while k != root:
        chain.append(k)
        k = int(m.body_parentid[k])
    p, q = np.zeros(3), np.array([1.0, 0, 0, 0])
    for k in reversed(chain):
        p = p + quat2mat(q) @ m.body_pos[k]
        q = quat_mul(q, m.body_quat[k])
    return p, q


@pytest.mark.parametrize("prec,tol", [("f64", 1e-12), ("f32", 1e-6)])
def test_tree_override_moves_the_welded_subtree(prec, tol):
    m = load("Lift_Panda")
    n = 4
    plain, sim = BatchedSim(m, n, precision=prec), BatchedSim(m, n, precision=prec)
    root = m.names["body"].index("robot0_base")
    sub = _welded_below(m, root)
    assert len(sub) == 6  # robot0_link0 and the five fixed_mount0_* bodies
    pos, quat = sim.body_pose_override_tree(root)
    rng = np.random.default_rng(0)
    P = pos.double().cpu().numpy() + rng.uniform(-0.2, 0.2, (n, 3))
    Q = rng.normal(size=(n, 4))
    Q /= np.linalg.norm(Q, axis=1, keepdims=True)
    pos.copy_(torch.as_tensor(P, dtype=pos.dtype))
    quat.copy_(torch.as_tensor(Q, dtype=quat.dtype))
    P, Q = pos.double().cpu().numpy(), quat.double().cpu().numpy()  # as the device holds them
    for s in (plain, sim):
        s.forward()
    xp, xq = sim.xpos.double().cpu().numpy(), sim.xquat.double().cpu().numpy()
    for e in range(n):
        for b in sub:
            lp, lq = _rel_pose(m, root, b)
            assert np.max(np.abs(xp[e, b] - (P[e] + quat2mat(Q[e]) @ lp))) < tol
            assert np.max(np.abs(xq[e, b] - quat_mul(Q[e], lq))) < tol
    # bodies outside the robot's tree are the plain handle's, bit for bit
    outside = [b for b in range(m.nbody) if int(m.body_rootid[b]) != root]
    assert outside
    assert torch.equal(sim.xpos[:, outside], plain.xpos[:, outside]) and torch.equal(sim.xquat[:, outside], plain.xquat[:, outside])
    plain.close()
    sim.close()


def test_tree_override_arguments():
    m = load("Lift_Panda")
    sim = BatchedSim(m, 2, precision="f64")
    L = lib()
    assert L.b2s_body_pose_override_tree(sim._h, 0) != 0
    assert L.b2s_body_pose_override_tree(sim._h, m.nbody) != 0
    with pytest.raises(B2SError):
        sim.body_pose_override_tree(m.names["body"].index("robot0_link1"))  # a moving body
    assert L.b2s_body_pose_override_tree(C.c_void_p(), 1) != 0
    sig0 = sim.snapshot_layout()[1]
    sim.body_pose_override_tree(m.names["body"].index("robot0_base"))
    assert sim.snapshot_layout()[1] != sig0
    sim.close()


SIZES = np.array([[0.8, 0.8, 0.05], [1.2, 0.7, 0.1], [0.6, 1.0, 0.03], [1.0, 0.9, 0.2]])
FRICTIONS = np.array([[1.0, 5e-3, 1e-4], [2.0, 1e-2, 2e-4], [1.5, 5e-3, 1e-4], [0.7, 5e-3, 1e-4]])


@pytest.mark.parametrize("field", ["size", "friction"])
def test_per_env_tables_match_batch_wide_tables(field):
    """environment e of a per-environment handle against a batch-wide handle built with environment e's table.  The per-environment
    handle recomputes the derived constants (invweights, mean inertia) on the device, the batch-wide one takes the compiler's: the
    two agree to rounding, so the trajectories agree to 1e-9 rather than bit for bit."""
    n = len(SIZES)
    kw = {"table_full_size": SIZES} if field == "size" else {"table_friction": FRICTIONS}
    per = _make(n=n, **kw)
    got = _rollout(per, 10)
    for e in range(n):
        one = {"table_full_size": SIZES[e]} if field == "size" else {"table_friction": FRICTIONS[e]}
        ref = _make(n=n, **one)
        want = _rollout(ref, 10)
        for x, y in zip(got, want):
            for u, v in zip(x, y):
                assert torch.max(torch.abs(u[e] - v[e])).item() < 1e-9
        ref.close()
    per.close()


def test_per_env_tables_are_independent_bit_for_bit():
    """each environment of a mixed per-environment handle equals the same environment of a handle whose every environment has
    its table, bit for bit (friction and size)"""
    n = len(SIZES)
    mixed = _rollout(_make(n=n, table_full_size=SIZES, table_friction=FRICTIONS), 10)
    for e in range(n):
        same = _rollout(_make(n=n, table_full_size=np.tile(SIZES[e], (n, 1)), table_friction=np.tile(FRICTIONS[e], (n, 1))), 10)
        for x, y in zip(mixed, same):
            for u, v in zip(x, y):
                assert torch.equal(u[e], v[e])


def test_schedules_agree_with_per_env_tables():
    """fused, pipeline and unit queue are bit-identical with per-environment tables, under the harness's settings (f32)"""
    from tests.schedules import make_env, random_actions, run

    res = []
    for mode in (0, 1, 2):
        env = make_env("Lift", len(SIZES), mode, 9, table_full_size=SIZES, table_friction=FRICTIONS)
        res.append(run(env, random_actions(env, 8), ("qpos", "obs")))
        env.close()
    for r in res[1:]:
        for a, b in zip(res[0], r):
            assert torch.equal(a, b)


def test_controller_follows_the_moved_base():
    """no contacts (the cube moved away): the eef trajectory relative to robot0_base is the same for two table lengths"""
    n = 2
    env = _make(n=n, table_full_size=np.array([[0.8, 0.8, 0.05], [1.4, 0.8, 0.05]]), initialization_noise=None)
    m = env.model
    base, site = m.names["body"].index("robot0_base"), env.eef_site_id
    q = env.sim.qpos.clone()
    q[:, env.cube_qadr:env.cube_qadr + 3] = torch.tensor([0.3, 0.35, 0.83], dtype=q.dtype)
    env.reset_to(q)
    env.sim.set_step1_export(True)
    a = torch.zeros((n, env.action_dim), dtype=env.dtype, device=env.device)
    a[:, :3] = torch.tensor([0.3, -0.2, 0.1], dtype=env.dtype)
    for _ in range(10):
        env.step(a)
        rel = (env.sim.site_xpos[:, site] - env.sim.xpos[:, base]).double()
        assert torch.max(torch.abs(rel[0] - rel[1])).item() < 1e-9
    assert abs(env.sim.xpos[1, base, 0].item() - (-0.16 - 0.7)) < 1e-15


def test_clone_and_masked_set_table():
    n = 6
    env = _make(n=n, table_full_size=np.tile(DEFAULT_SIZE, (n, 1)), table_friction=np.tile(DEFAULT_FRICTION, (n, 1)))
    mask = torch.zeros(n, dtype=torch.bool, device=env.device)
    mask[1] = mask[4] = True
    before = env.sim.snapshot()
    env.set_table(full_size=(1.2, 0.6, 0.1), friction=(2.0, 5e-3, 1e-4), mask=mask)
    env.reset(mask=mask)
    after = env.sim.snapshot()
    for name in ("geom_size:%d" % env.model.names["geom"].index("table_collision"), "qpos", "qvel"):
        x, y = before.field(name), after.field(name)
        assert torch.equal(x[~mask], y[~mask]), name
    assert np.allclose(env.table_full_size[1], [1.2, 0.6, 0.1]) and np.allclose(env.table_full_size[0], DEFAULT_SIZE)
    assert abs(env.sim.xpos[4, env.model.names["body"].index("robot0_base"), 0].item() - (-0.76)) < 1e-15
    env.clone_envs([0, 1, 2, 3, 4, 1])  # environment 5 continues from environment 1, table included
    t = env.model.names["geom"].index("table_collision")
    assert torch.equal(env.sim.array("geom_size:%d" % t)[5], env.sim.array("geom_size:%d" % t)[1])
    for a in _actions(env, 10):
        a[5] = a[1]
        env.step(a)
    assert torch.equal(env.sim.qpos[1], env.sim.qpos[5]) and torch.equal(env.flat_obs()[1], env.flat_obs()[5])
    env.close()
