"""Per-environment model values (b2s_model_override / b2s_set_const): geom sizes and friction, body masses and moments per
environment, with the constants derived from them (dof_invweight0, body_invweight0, meaninertia, geom bounds) computed on the device.
Every environment is checked against an oracle built from its own overridden host model (tests/model_override_host.py)."""
import glob
import os

import numpy as np
import pytest

from tests.model_override_host import override_model
from tests.schedules import make_env, random_actions, run
from tests.util import ROOT, lift_states, load

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

PACKAGED = sorted(glob.glob(os.path.join(ROOT, "robosuite_b200", "assets", "models", "*.npz")))
QPOS_OBS = ("qpos", "obs")  # what the schedule and masking comparisons here hold bit-identical


def _free_bodies(m):
    """the free-floating objects (Door has none: its last moving body, the latch, stands in)"""
    free = [int(m.jnt_bodyid[j]) for j in range(m.njnt) if int(m.jnt_type[j]) == 0]
    return free or [max(b for b in range(m.nbody) if int(m.body_weldid[b]) != 0)]


def _rel(a, b):
    """elementwise relative error (exact zeros must stay exact)"""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    nz = b != 0
    assert np.all(a[~nz] == 0)
    return float(np.max(np.abs(a[nz] - b[nz]) / np.abs(b[nz]))) if nz.any() else 0.0


@pytest.mark.parametrize("prec,tol", [("f64", 1e-12), ("f32", 1e-4)])
def test_set_const_matches_compiler_on_every_packaged_model(prec, tol):
    from robosuite_b200.engine import BatchedSim
    from robosuite_b200.mjcf.compiler import load_model

    worst = {}
    for path in PACKAGED:
        m = load_model(path)
        n = 3
        sim = BatchedSim(m, n, precision=prec)
        bodies = _free_bodies(m)
        views = {b: (sim.model_override("body_mass", b), sim.model_override("body_inertia", b)) for b in bodies}
        sim.set_const()
        got = [sim.body_invweight0.cpu().numpy(), sim.dof_invweight0.cpu().numpy(), sim.meaninertia.cpu().numpy()]
        for e in range(n):  # the model's own values: the compiler's constants
            for k, (g, ref) in enumerate(zip(got, (m.body_invweight0, m.dof_invweight0, m.stat_meaninertia))):
                worst[(os.path.basename(path), k, "model")] = _rel(g[e], ref)
        # env 1: masses and moments x 0.5, env 2: x 3
        for e, f in ((1, 0.5), (2, 3.0)):
            for b, (mv, iv) in views.items():
                mv[e] = mv[e] * f
                iv[e] = iv[e] * f
        sim.set_const()
        got = [sim.body_invweight0.cpu().numpy(), sim.dof_invweight0.cpu().numpy(), sim.meaninertia.cpu().numpy()]
        for e, f in ((1, 0.5), (2, 3.0)):
            h = override_model(m, body_mass={b: m.body_mass[b] * f for b in bodies},
                               body_inertia={b: m.body_inertia[b] * f for b in bodies})
            for k, (g, ref) in enumerate(zip(got, (h.body_invweight0, h.dof_invweight0, h.stat_meaninertia))):
                worst[(os.path.basename(path), k, f)] = _rel(g[e], ref)
        assert int(sim.warn.abs().max()) == 0
        sim.close()
    print(prec, "max relative error %.3g" % max(worst.values()))
    bad = {k: v for k, v in worst.items() if v > tol}
    assert not bad, bad


def _cube(m):
    return m.names["geom"].index("cube_g0"), m.names["body"].index("cube_main")


def _box_inertia(m, g, b, s):
    from robosuite_b200.mjcf.compiler import quat2mat

    mass = 8000.0 * np.prod(s)
    box = mass / 3 * np.array([s[1] ** 2 + s[2] ** 2, s[0] ** 2 + s[2] ** 2, s[0] ** 2 + s[1] ** 2])
    W = (quat2mat(m.body_iquat[b]).T @ quat2mat(m.geom_quat[g])) ** 2
    return mass, W @ box


def _per_env_cubes(m, n, seed=3):
    """env 0: the model's own cube; the others: sizes, masses (density 1000) and frictions of their own"""
    g, b = _cube(m)
    rng = np.random.default_rng(seed)
    out = []
    for e in range(n):
        if e == 0:
            out.append((m.geom_size[g].copy(), m.geom_friction[g].copy(), float(m.body_mass[b]), m.body_inertia[b].copy()))
            continue
        s = rng.uniform(0.017, 0.026, 3)
        mass, inertia = _box_inertia(m, g, b, s)
        fr = m.geom_friction[g] * rng.uniform(0.5, 1.5, 3)
        out.append((s, fr, mass, inertia))
    return out


def _sim_with_cubes(m, n, prec, cubes, **kw):
    from robosuite_b200.engine import BatchedSim

    g, b = _cube(m)
    sim = BatchedSim(m, n, precision=prec, **kw)
    sz, fr = sim.model_override("geom_size", g), sim.model_override("geom_friction", g)
    ms, ine = sim.model_override("body_mass", b), sim.model_override("body_inertia", b)
    for e, (s, f, mass, inertia) in enumerate(cubes):
        sz[e] = torch.as_tensor(s); fr[e] = torch.as_tensor(f); ms[e] = mass; ine[e] = torch.as_tensor(inertia)
    sim.set_const()
    return sim


def _oracle_for(m, cube):
    from oracle.pyoracle import Oracle
    from robosuite_b200.mjcf.compiler import pack_model

    g, b = _cube(m)
    s, f, mass, inertia = cube
    return Oracle(pack_model(override_model(m, geom_size={g: s}, geom_friction={g: f}, body_mass={b: mass}, body_inertia={b: inertia})))


@pytest.mark.parametrize("prec", ["f64", "f32"])
def test_per_environment_cubes_follow_their_own_oracles(prec):
    """8 Lift environments with different cubes: the gripper closes while the arm pushes down and then up with the cube between
    the fingers or resting beside them; every environment against the oracle of its own model, substep by substep"""
    m = load("Lift_Panda")
    n, nsub = 8, 100
    cubes = _per_env_cubes(m, n)
    q, _ = lift_states(m, n, seed=4)
    for e in range(n):
        q[e, 11] = 0.8 + cubes[e][0][2] + 5e-4  # each cube starts just above the table, its own half height
    sim = _sim_with_cubes(m, n, prec, cubes)
    dt = sim.dtype
    sim.qpos.copy_(torch.as_tensor(q, dtype=dt))
    rng = np.random.default_rng(6)
    ctrl = np.zeros((n, m.nu))
    ctrl[:, :7] = rng.uniform(-3, 3, size=(n, 7)) + np.array([0, -4, 0, -20, 0, 2, 0])
    ctrl[:, 7:9] = [0.0, 0.0]  # close the gripper
    oracles = [_oracle_for(m, c) for c in cubes]
    for e, o in enumerate(oracles):
        o.qpos[:] = q[e]; o.ctrl[:] = ctrl[e]
    eq = ev = 0.0
    for t in range(nsub):
        c = ctrl.copy()
        c[:, 1] += 6.0 if t >= nsub // 2 else 0.0  # lift phase
        sim.ctrl.copy_(torch.as_tensor(c, dtype=dt))
        sim.step2()
        torch.cuda.synchronize()
        cg, nc, ne = sim.contact_geom.cpu().numpy(), sim.ncon.cpu().numpy(), sim.nefc.cpu().numpy()
        for e, o in enumerate(oracles):
            o.ctrl[:] = c[e]
            o.step()
            oc = o.contacts()
            assert int(nc[e]) == len(oc), (t, e)
            assert [(int(a), int(b)) for a, b in cg[e][: len(oc)]] == [(x["geom1"], x["geom2"]) for x in oc], (t, e)
            assert int(ne[e]) == o.nefc, (t, e)
    qd, vd = sim.qpos.cpu().numpy().astype(np.float64), sim.qvel.cpu().numpy().astype(np.float64)
    for e, o in enumerate(oracles):
        eq = max(eq, np.abs(qd[e] - o.qpos).max() / max(np.abs(o.qpos).max(), 1e-9))
        ev = max(ev, np.abs(vd[e] - o.qvel).max() / max(np.abs(o.qvel).max(), 1e-9))
    print(prec, "per-environment cubes: rel err qpos %.3g qvel %.3g" % (eq, ev))
    if prec == "f64":
        assert eq < 1e-7 and ev < 1e-6
    else:
        assert eq < 1e-4 and ev < 1e-4
    assert int(sim.warn.abs().max()) == 0
    sim.close()


@pytest.mark.parametrize("prec", ["f64", "f32"])
def test_enlarged_cube_rests_on_the_table(prec):
    """a 0.05 half-size cube: the model's bounding radius (0.036) would cull its plane and table pairs, so it only stays up when the
    derived bounds are per environment"""
    m = load("Lift_Panda")
    g, b = _cube(m)
    s = np.full(3, 0.05)
    mass, inertia = _box_inertia(m, g, b, s)
    cubes = [(s, m.geom_friction[g], mass, inertia)] * 2
    sim = _sim_with_cubes(m, 2, prec, cubes)
    assert float(sim.array("geom_rbound:%d" % g)[0]) > 0.08
    q, _ = lift_states(m, 2, seed=1)
    q[:, 9:11] = [[0.25, 0.25], [0.25, -0.25]]  # out of the arm's way
    top = 0.8  # table top
    q[:, 11] = top + 0.05
    sim.qpos.copy_(torch.as_tensor(q, dtype=sim.dtype))
    ctrl = np.zeros((2, m.nu))
    ctrl[:, :7] = [0, -4, 0, -20, 0, 2, 0]
    sim.ctrl.copy_(torch.as_tensor(ctrl, dtype=sim.dtype))
    o = _oracle_for(m, cubes[0])
    o.qpos[:] = q[0]; o.ctrl[:] = ctrl[0]
    zs = []
    for _ in range(100):
        sim.step(1)
        o.step()
        zs.append(sim.qpos[:, 11].cpu().numpy().astype(np.float64))
    zs = np.array(zs)
    print(prec, "enlarged cube: max |z - (table + 0.05)| = %.3g" % np.abs(zs - (top + 0.05)).max())
    assert np.abs(zs - (top + 0.05)).max() < 1e-3
    assert abs(zs[-1, 0] - o.qpos[11]) < (1e-9 if prec == "f64" else 1e-4)
    sim.close()


@pytest.mark.parametrize("tier", [None, (4, 16)])
def test_schedules_agree_with_overrides(tier):
    """fused, pipeline and unit queue are bit-identical with per-environment cubes; (4, 16) forces environments into the large tier"""
    n = 64
    res = []
    for mode in (0, 1, 2):
        kw = {"tier_small": tier} if tier else {}
        env = make_env("Lift", n, mode, 9, per_env_cube_size=True, hard_reset=True, **kw)
        acts = random_actions(env, 8)
        res.append(run(env, acts, QPOS_OBS))
        mask = torch.zeros(n, dtype=torch.bool, device=env.device)
        mask[::5] = True
        env.reset(mask=mask)  # new cubes for the masked environments
        res[-1] = res[-1] + run(env, acts[:4], QPOS_OBS)
        env.close()
    for r in res[1:]:
        for a, b in zip(res[0], r):
            assert torch.equal(a, b)


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_declaring_overrides_changes_no_bit(mode):
    n = 32
    a, b = make_env("Lift", n, mode, 9), make_env("Lift", n, mode, 9)
    m = a.model
    g, body = _cube(m)
    for gg in (g, m.names["geom"].index("table_collision")):
        b.sim.model_override("geom_size", gg)
        b.sim.model_override("geom_friction", gg)
    b.sim.model_override("body_mass", body)
    b.sim.model_override("body_inertia", body)
    acts = random_actions(a, 10)
    ra, rb = run(a, acts, QPOS_OBS), run(b, acts, QPOS_OBS)
    for x, y in zip(ra, rb):
        assert torch.equal(x, y)
    a.close()
    b.close()


def test_masked_reset_with_new_cubes_leaves_the_others_alone():
    n = 64
    a = make_env("Lift", n, 1, 5, per_env_cube_size=True, hard_reset=True)
    b = make_env("Lift", n, 1, 5, per_env_cube_size=True, hard_reset=True)
    acts = random_actions(a, 10)
    run(a, acts[:5]); run(b, acts[:5])
    mask = torch.zeros(n, dtype=torch.bool, device=a.device)
    mask[3::7] = True
    size = a._cube_ov[0]
    before = {k: getattr(a.sim, k).clone() for k in ("qpos", "qvel", "obs", "ctrl_goal_pos")}
    s0 = size.clone()
    a.reset(mask=mask)
    assert torch.equal(size[~mask], s0[~mask]) and not torch.equal(size[mask], s0[mask])
    for k, v in before.items():
        assert torch.equal(getattr(a.sim, k)[~mask], v[~mask]), k
    ra, rb = run(a, acts[5:], QPOS_OBS), run(b, acts[5:], QPOS_OBS)
    for x, y in zip(ra, rb):
        assert torch.equal(x[~mask], y[~mask])
    assert int(a.sim.warn.abs().max()) == 0


def test_lift_per_env_cube_size():
    n = 64
    env = make_env("Lift", n, 1, 2, per_env_cube_size=True, hard_reset=True)
    m = env.model
    g, b = _cube(m)
    size, mass, inertia = (t.double().cpu().numpy() for t in env._cube_ov)
    assert size.min() >= 0.020 and size.max() <= 0.022 and len(np.unique(size[:, 0])) == n
    for e in range(n):
        mm, ii = _box_inertia(m, g, b, size[e])
        assert abs(mass[e] - mm) <= 1e-6 * mm and np.allclose(inertia[e], ii, rtol=1e-6)
    assert np.allclose(env.sim.qpos[:, env.cube_qadr + 2].double().cpu().numpy(), 0.81 + size[:, 2], atol=1e-6)
    zero = torch.zeros((n, env.action_dim), device=env.device, dtype=env.dtype)
    for _ in range(20):
        env.step(zero)
    v = env.sim.qvel[:, m.jnt_dofadr[env.cube_joint]:m.jnt_dofadr[env.cube_joint] + 6].abs().max()
    assert float(v) < 1e-2, float(v)
    mask = torch.zeros(n, dtype=torch.bool, device=env.device)
    mask[::3] = True
    s0 = env._cube_ov[0].clone()
    env.reset(mask=mask)
    s1 = env._cube_ov[0]
    assert torch.equal(s1[~mask], s0[~mask]) and bool((s1[mask] != s0[mask]).all())
    assert int(env.sim.warn.abs().max()) == 0
    # without hard_reset the cubes are drawn once
    env2 = make_env("Lift", 8, 1, 2, per_env_cube_size=True)
    s0 = env2._cube_ov[0].clone()
    env2.reset()
    assert torch.equal(env2._cube_ov[0], s0)
    env.close()
    env2.close()


def test_errors_and_invalid_values():
    from robosuite_b200.engine import B2SError, BatchedSim
    from robosuite_b200.mjcf.compiler import GEOM_MESH, GEOM_PLANE

    m = load("Lift_Panda")
    sim = BatchedSim(m, 4, precision="f32")
    L, h = sim._L, sim._h
    cg = set()
    for p in m.pair_geom:
        cg.update(int(x) for x in p)
    mesh = next(i for i in cg if int(m.geom_type[i]) == GEOM_MESH)
    plane = next(i for i in cg if int(m.geom_type[i]) == GEOM_PLANE)
    vis = m.names["geom"].index("cube_g0_vis")
    assert vis not in cg
    for f, i in (("geom_size", mesh), ("geom_size", plane), ("geom_friction", vis), ("body_mass", 0)):
        assert L.b2s_model_override(h, f.encode(), i) == -4, (f, i)
    assert L.b2s_model_override(h, b"geom_solref", 88) == -1
    assert L.b2s_model_override(h, b"geom_size", m.ngeom) == -1
    assert L.b2s_model_override(h, b"body_mass", -1) == -1
    moving = [b for b in range(1, m.nbody) if int(m.body_weldid[b]) != 0]
    for b in moving[:8]:
        sim.model_override("body_mass", b)
    assert L.b2s_model_override(h, b"body_mass", moving[8]) == -4
    with pytest.raises(B2SError):
        sim.model_override("body_inertia", moving[8])
    sim.close()
    sim = BatchedSim(m, 4, precision="f32")
    g, b = _cube(m)
    size, mass, inertia = sim.model_override("geom_size", g), sim.model_override("body_mass", b), sim.model_override("body_inertia", b)
    size[1, 0] = -0.01
    mass[2] = float("nan")
    inertia[3] = torch.tensor([1e-5, 1e-5, 3e-5])
    sim.set_const()
    assert sim.warn.cpu().tolist() == [0, 128, 128, 128]
    sim.close()
    # the geom cap: nine colliding primitive geoms in one model
    from robosuite_b200.mjcf.compiler import load_model

    for path in PACKAGED:
        pm = load_model(path)
        prim = sorted({int(x) for p in pm.pair_geom for x in p if int(pm.geom_type[int(x)]) in (2, 3, 4, 5, 6)})
        if len(prim) > 8:
            s2 = BatchedSim(pm, 2, precision="f32")
            for gg in prim[:8]:
                s2.model_override("geom_size", gg)
            assert s2._L.b2s_model_override(s2._h, b"geom_size", prim[8]) == -4
            s2.close()
            break
    else:
        pytest.fail("no packaged model has nine colliding primitive geoms")
