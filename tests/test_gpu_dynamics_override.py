"""Per-environment joint damping, armature, friction loss and contact solref / solimp (b2s_model_override), the device perturbation
(b2s_perturb_config / b2s_perturb_model) and BatchedDomainRandomizationWrapper.  Every environment is checked against an oracle
built from its own host model (tests/dynamics_override_host.py), the draws against the numpy restatement of the kernel."""
import glob
import os

import numpy as np
import pytest

from tests.dynamics_override_host import dynamics_override_model, perturb_values
from tests.schedules import make_env, random_actions, run
from tests.util import ROOT, load

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

PACKAGED = sorted(glob.glob(os.path.join(ROOT, "robosuite_b200", "assets", "models", "*.npz")))
DOF = ("dof_damping", "dof_armature", "dof_frictionloss")


def _rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    nz = b != 0
    assert np.all(a[~nz] == 0)
    return float(np.max(np.abs(a[nz] - b[nz]) / np.abs(b[nz]))) if nz.any() else 0.0


@pytest.mark.parametrize("prec,tol", [("f64", 1e-12), ("f32", 1e-4)])
def test_set_const_with_per_environment_armature_matches_the_compiler(prec, tol):
    from robosuite_b200.engine import BatchedSim
    from robosuite_b200.mjcf.compiler import load_model

    worst = {}
    for path in PACKAGED:
        m = load_model(path)
        sim = BatchedSim(m, 3, precision=prec)
        arm = sim.model_override("dof_armature")
        for e, f in ((1, 0.5), (2, 3.0)):
            arm[e] = torch.as_tensor(m.dof_armature * f + 0.01 * f, dtype=sim.dtype)
        sim.set_const()
        got = [sim.body_invweight0.cpu().numpy(), sim.dof_invweight0.cpu().numpy(), sim.meaninertia.cpu().numpy()]
        for k, ref in enumerate((m.body_invweight0, m.dof_invweight0, m.stat_meaninertia)):
            worst[(os.path.basename(path), k, 1.0)] = _rel(got[k][0], ref)
        for e, f in ((1, 0.5), (2, 3.0)):
            h = dynamics_override_model(m, dof_armature={-1: m.dof_armature * f + 0.01 * f})
            for k, ref in enumerate((h.body_invweight0, h.dof_invweight0, h.stat_meaninertia)):
                worst[(os.path.basename(path), k, f)] = _rel(got[k][e], ref)
        assert int(sim.warn.abs().max()) == 0
        sim.close()
    print(prec, "armature: max relative error %.3g" % max(worst.values()))
    bad = {k: v for k, v in worst.items() if v > tol}
    assert not bad, bad


def _object_geoms(m):
    """colliding primitive geoms of the moving bodies outside the robot and the gripper (at most 8)"""
    bn = m.names["body"]
    mov = {b for b in range(1, m.nbody) if int(m.body_weldid[b]) != 0 and not bn[b].startswith(("robot0_", "gripper0_"))}
    cg = {int(g) for p in m.pair_geom for g in p}
    return [g for g in range(m.ngeom) if int(m.geom_bodyid[g]) in mov and g in cg and int(m.geom_type[g]) in (2, 3, 4, 5, 6)][:8]


def _per_env_values(m, n, seed=12):
    """env 0: the model's values; the others their own damping, armature, friction loss and object solref / solimp.  Env 1 adds
    friction loss to the free joints' dofs (rows the model does not have), env 2 drops the friction loss of arm dof 3 (a row the model
    has).  The comparison is bit-level: an object corner whose contact distance crosses zero slowly makes the substep of the crossing
    depend on the last bit, where the engine and the oracle may differ and both be right.  Seed 11 has such a crossing (Lift env 7 near
    substep 70, Stack env 5 near substep 90, with or without arm motion); seed 12 has none within the 100 substeps."""
    rng = np.random.default_rng(seed)
    geoms = _object_geoms(m)
    free = [d for j in range(m.njnt) if int(m.jnt_type[j]) == 0 for d in range(int(m.jnt_dofadr[j]), int(m.jnt_dofadr[j]) + 6)]
    out = []
    for e in range(n):
        v = {"dof_damping": {-1: m.dof_damping.copy()}, "dof_armature": {-1: m.dof_armature.copy()},
             "dof_frictionloss": {-1: m.dof_frictionloss.copy()},
             "geom_solref": {g: m.geom_solref[g].copy() for g in geoms}, "geom_solimp": {g: m.geom_solimp[g].copy() for g in geoms}}
        if e > 0:
            v["dof_damping"][-1] = m.dof_damping * rng.uniform(0.5, 1.5, m.nv) + rng.uniform(0, 0.02, m.nv)
            v["dof_armature"][-1] = m.dof_armature * rng.uniform(0.5, 2.0, m.nv) + rng.uniform(0, 0.02, m.nv)
            v["dof_frictionloss"][-1] = m.dof_frictionloss * rng.uniform(0.5, 1.5, m.nv)
            for g in geoms:
                v["geom_solref"][g] = m.geom_solref[g] * rng.uniform(0.8, 1.5, 2)
                v["geom_solimp"][g] = m.geom_solimp[g] * np.r_[rng.uniform(0.95, 1.0, 2), rng.uniform(0.5, 2.0), 1, 1]
        if e == 1 and free:
            v["dof_frictionloss"][-1][free] = 0.02
        if e == 2:
            v["dof_frictionloss"][-1][3] = 0.0
        out.append(v)
    return out


def _task_model_and_states(task, n, seed=3):
    """the task's model (Door: its door placed where the task places it by default) and reset states of n environments"""
    import robosuite_b200 as suite

    env = suite.make(task, robots="Panda", num_envs=n, seed=seed, **({"door_placement": (0.08, 0.0, -np.pi / 2 - 0.125)} if task == "Door" else {}))
    m, q = env.model, env._reset_qpos.double().cpu().numpy().copy()
    env.close()
    # every free object starts 0.5 mm above the table top instead of the task's 10 mm: a short landing, not a tumble whose corner
    # contacts come and go on last-bit differences
    geoms = _object_geoms(m)
    for j in range(m.njnt):
        if int(m.jnt_type[j]) == 0:
            g = next(g for g in geoms if int(m.geom_bodyid[g]) == int(m.jnt_bodyid[j]))
            q[:, int(m.jnt_qposadr[j]) + 2] = 0.8 + m.geom_size[g, 2] + 5e-4
    return m, q


@pytest.mark.parametrize("task", ["Lift", "Stack", "Door"])
@pytest.mark.parametrize("prec", ["f64", "f32"])
def test_per_environment_dynamics_follow_their_own_oracles(task, prec):
    from oracle.pyoracle import Oracle
    from robosuite_b200.engine import BatchedSim
    from robosuite_b200.mjcf.compiler import pack_model

    n, nsub = 8, 100
    m, q = _task_model_and_states(task, n)
    vals = _per_env_values(m, n)
    sim = BatchedSim(m, n, precision=prec, maxefc=max(m.nv + 8, 128))
    dt = sim.dtype
    for f in ("dof_damping", "dof_armature", "dof_frictionloss", "geom_solref", "geom_solimp"):
        for i in vals[0][f]:
            t = sim.model_override(f, None if f in DOF else i)
            for e in range(n):
                t[e] = torch.as_tensor(vals[e][f][i], dtype=dt)
    sim.set_const()
    sim.qpos.copy_(torch.as_tensor(q, dtype=dt))
    rng = np.random.default_rng(6)
    ctrl = np.zeros((n, m.nu))
    ctrl[:, :7] = rng.uniform(-1, 1, size=(n, 7)) + np.array([0, 2, 0, -20, 0, 2, 0])
    oracles = [Oracle(pack_model(dynamics_override_model(m, **vals[e]))) for e in range(n)]
    for e, o in enumerate(oracles):
        o.qpos[:] = q[e]
    # the shoulder lifts the arm away while the objects land on the table: no grasp and no finger-table impact, whose first contact
    # points can differ between the engine and the oracle on a last-bit difference (both are right; the comparison would end there)
    for t in range(nsub):
        c = ctrl
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
    eq = max(np.abs(qd[e] - o.qpos).max() / max(np.abs(o.qpos).max(), 1e-9) for e, o in enumerate(oracles))
    ev = max(np.abs(vd[e] - o.qvel).max() / max(np.abs(o.qvel).max(), 1e-9) for e, o in enumerate(oracles))
    print(task, prec, "per-environment dynamics: rel err qpos %.3g qvel %.3g" % (eq, ev))
    tol = 1e-12 if prec == "f64" else 1e-4
    assert eq <= tol and ev <= tol
    assert int(sim.warn.abs().max()) == 0
    sim.close()


@pytest.mark.parametrize("tier", [None, (4, 16)])
def test_schedules_agree_with_randomized_dynamics(tier):
    """fused, pipeline and unit queue are bit-identical with every field randomised per environment; (4, 16) forces environments
    into the large tier"""
    from robosuite_b200.wrappers import BatchedDomainRandomizationWrapper

    n = 64
    res = []
    for mode in (0, 1, 2):
        env = make_env("Lift", n, mode, 9, **({"tier_small": tier} if tier else {}))
        w = BatchedDomainRandomizationWrapper(env, seed=5, randomize_every_n_steps=3)
        w.reset()
        acts = random_actions(env, 8)
        r = run(w, acts)
        mask = torch.zeros(n, dtype=torch.bool, device=env.device)
        mask[::5] = True
        w.reset(mask=mask)
        res.append(r + run(w, acts[:4]) + (env.sim.model_override("dof_frictionloss").clone(),))
        env.close()
    for r in res[1:]:
        for a, b in zip(res[0], r):
            assert torch.equal(a, b)


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_declaring_dynamics_overrides_changes_no_bit(mode):
    n = 32
    a, b = make_env("Lift", n, mode, 9), make_env("Lift", n, mode, 9)
    m = a.model
    for f in DOF:
        b.sim.model_override(f)
    for g in (m.names["geom"].index("cube_g0"), m.names["geom"].index("table_collision")):
        b.sim.model_override("geom_solref", g)
        b.sim.model_override("geom_solimp", g)
    acts = random_actions(a, 10)
    ra, rb = run(a, acts), run(b, acts)
    for x, y in zip(ra, rb):
        assert torch.equal(x, y)
    a.close()
    b.close()


def test_masked_perturbation_and_reset_leave_the_others_alone():
    from robosuite_b200.wrappers import BatchedDomainRandomizationWrapper

    n = 64
    a, b = make_env("Lift", n, 1, 5), make_env("Lift", n, 1, 5)
    wa = BatchedDomainRandomizationWrapper(a, seed=1, randomize_every_n_steps=0)
    wb = BatchedDomainRandomizationWrapper(b, seed=1, randomize_every_n_steps=0)
    acts = random_actions(a, 10)
    run(wa, acts[:5]); run(wb, acts[:5])
    mask = torch.zeros(n, dtype=torch.bool, device=a.device)
    mask[3::7] = True
    damp = a.sim.model_override("dof_damping")
    d0 = damp.clone()
    before = {k: getattr(a.sim, k).clone() for k in ("qpos", "qvel", "obs", "ctrl_goal_pos", "dof_invweight0", "meaninertia")}
    wa.reset(mask=mask)
    torch.cuda.synchronize()
    assert torch.equal(damp[~mask], d0[~mask]) and not torch.equal(damp[mask], d0[mask])
    for k, v in before.items():
        assert torch.equal(getattr(a.sim, k)[~mask], v[~mask]), k
    ra, rb = run(wa, acts[5:]), run(wb, acts[5:])
    for x, y in zip(ra, rb):
        assert torch.equal(x[~mask], y[~mask])
    assert int(a.sim.warn.abs().max()) == 0


def _perturb_sim(n, prec="f64"):
    from robosuite_b200.engine import BatchedSim

    m = load("Lift_Panda")
    g, b = m.names["geom"].index("cube_g0"), m.names["body"].index("cube_main")
    sim = BatchedSim(m, n, precision=prec)
    spec = [("body_mass", b, "scale", 0.3), ("body_inertia", b, "scale", 0.2, True), ("geom_friction", g, "scale", 0.1),
            ("geom_solref", g, "scale", 0.1), ("geom_solimp", g, "scale", 0.05), ("geom_size", g, "scale", 0.1),
            ("dof_damping", None, "shift", 0.05), ("dof_armature", 2, "shift", 0.5), ("dof_frictionloss", None, "shift", 0.05)]
    for f, i, *_ in spec:
        sim.model_override(f, None if f in DOF else i)
    sim.perturb_config(spec)
    return m, sim, spec


def _device_values(sim, spec):
    out = []
    for f, i, *_ in spec:
        t = sim.model_override(f, None if f in DOF else i).double().cpu().numpy()
        out.append(t[:, i:i + 1] if f in DOF and i is not None else (t[:, None] if t.ndim == 1 else t))
    return out


@pytest.mark.parametrize("prec", ["f64", "f32"])
def test_perturbation_draws_match_the_host_restatement(prec):
    m, sim, spec = _perturb_sim(64, prec)
    mask = torch.zeros(64, dtype=torch.uint8, device=sim.torch_device)
    mask[1::3] = 1
    before = _device_values(sim, spec)
    sim.perturb_model(mask, seed=2 ** 40 + 17, counter=5)
    torch.cuda.synchronize()
    got = _device_values(sim, spec)
    sel = mask.bool().cpu().numpy()
    ref = perturb_values(m, spec, np.nonzero(sel)[0], 2 ** 40 + 17, 5)
    npdt = np.float64 if prec == "f64" else np.float32
    for k in range(len(spec)):
        assert np.array_equal(got[k][sel], ref[k].astype(npdt).astype(np.float64)), spec[k]
        assert np.array_equal(got[k][~sel], before[k][~sel]), spec[k]
    # repeated calls draw around the model's value again: no random walk
    sim.perturb_model(None, seed=3, counter=0)
    sim.perturb_model(None, seed=3, counter=0)
    ref = perturb_values(m, spec, range(64), 3, 0)
    for k, v in enumerate(_device_values(sim, spec)):
        assert np.array_equal(v, ref[k].astype(npdt).astype(np.float64))
    sim.close()


def test_perturbation_draws_do_not_depend_on_the_batch():
    m, a, spec = _perturb_sim(4)
    _, b, _ = _perturb_sim(64)
    for s in (a, b):
        s.perturb_model(None, seed=77, counter=3)
    torch.cuda.synchronize()
    for x, y in zip(_device_values(a, spec), _device_values(b, spec)):
        assert np.array_equal(x, y[:4])
    a.close()
    b.close()


def test_perturbation_bounds_and_statistics():
    from robosuite_b200.engine import BatchedSim

    m = load("Lift_Panda")
    g, b = m.names["geom"].index("cube_g0"), m.names["body"].index("cube_main")
    n, a = 4096, 0.3
    sim = BatchedSim(m, n, precision="f64")
    sim.model_override("body_mass", b)
    sim.model_override("dof_damping")
    sim.model_override("body_inertia", b)
    sim.perturb_config([("body_mass", b, "scale", a), ("dof_damping", None, "shift", 0.05), ("body_inertia", b, "scale", a, True)])
    sim.perturb_model(None, seed=12345, counter=0)
    torch.cuda.synchronize()
    d = sim.model_override("body_mass", b).cpu().numpy() / m.body_mass[b] - 1
    assert np.all(np.abs(d) <= a)
    sd = a / np.sqrt(3)  # U(-a, a)
    assert abs(d.mean()) < 4 * sd / np.sqrt(n)
    assert abs(d.std() - sd) < 4 * sd / np.sqrt(2 * n) * 1.2
    damp = sim.model_override("dof_damping").cpu().numpy()
    assert np.all(damp >= 0) and np.all(damp <= m.dof_damping + 0.05)
    zero = m.dof_damping == 0
    frac = (damp[:, zero] == 0).mean()  # shift mode clipped at 0: half of the draws of a zero-damping dof
    assert abs(frac - 0.5) < 4 * 0.5 / np.sqrt(n * zero.sum())
    ine = sim.model_override("body_inertia", b).cpu().numpy() / m.body_inertia[b]
    assert np.allclose(ine, ine[:, :1], rtol=1e-13)
    sim.close()


def _staggered_gym(n, k, horizon):
    import robosuite_b200 as suite
    from robosuite_b200.wrappers import BatchedDomainRandomizationWrapper, BatchedGymWrapper

    env = suite.make("Lift", robots="Panda", num_envs=n, seed=4, horizon=horizon)
    w = BatchedDomainRandomizationWrapper(env, seed=8, randomize_every_n_steps=k)
    gym = BatchedGymWrapper(w)
    gym.reset()
    env.set_episode_steps(np.arange(n) % horizon)
    return env, gym


@pytest.mark.parametrize("k", [0, 3])
def test_gym_auto_reset_randomizes_the_finished_environments(k):
    """two horizons with staggered episode clocks: at an auto-reset only the finished environments' arrays change; with
    randomize_every_n_steps=k also those whose clock is a multiple of k before the step"""
    n, horizon = 16, 7
    env, gym = _staggered_gym(n, k, horizon)
    arrays = [env.sim.model_override("dof_damping"), env.sim.model_override("body_mass", env.cube_body_id),
              env.sim.model_override("geom_solimp", env.model.names["geom"].index("cube_g0"))]
    zero = np.zeros((n, env.action_dim), dtype=np.float32)
    changed_any = 0
    for _ in range(2 * horizon):
        clocks = env.timestep.clone()
        before = [a.clone() for a in arrays]
        _, _, term, _, _ = gym.step(zero)
        torch.cuda.synchronize()
        finished = term.bool()
        due = (clocks % k == 0) if k else torch.zeros_like(finished)
        expect = finished | due
        for a, a0 in zip(arrays, before):
            diff = (a != a0).reshape(n, -1).any(dim=1)
            assert torch.equal(diff & ~expect, torch.zeros_like(diff))
            assert bool(diff[expect].all())
        changed_any += int(finished.sum())
    assert changed_any >= n  # every environment finished at least once
    assert int(env.sim.warn.abs().max()) == 0
    env.close()


def test_errors_and_invalid_values():
    from robosuite_b200.engine import B2SError, BatchedSim
    from robosuite_b200.mjcf.compiler import GEOM_MESH

    m = load("Lift_Panda")
    sim = BatchedSim(m, 4, precision="f32")
    L, h = sim._L, sim._h
    cg = {int(x) for p in m.pair_geom for x in p}
    mesh = next(i for i in cg if int(m.geom_type[i]) == GEOM_MESH)
    assert L.b2s_model_override(h, b"dof_damping", 0) == -1
    assert L.b2s_model_override(h, b"dof_armature", 3) == -1
    # solref / solimp are no fields of their own: they come with a declared geom's slot
    g = m.names["geom"].index("cube_g0")
    assert L.b2s_model_override(h, b"geom_solref", g) == -1
    assert L.b2s_model_override(h, b"geom_solimp", g) == -1
    for f in ("geom_solref", "geom_solimp"):  # a mesh has no slot, so no per-environment solref / solimp
        with pytest.raises(B2SError):
            sim.model_override(f, mesh)
    assert L.b2s_model_override(h, b"geom_friction", mesh) == -4
    damp, solimp = sim.model_override("dof_damping"), sim.model_override("geom_solimp", g)
    assert sim.array("geom_solref:%d" % g).shape == (4, 2)  # the same slot carries solref
    table = m.names["geom"].index("table_collision")
    from robosuite_b200.engine import PerturbSpec

    def cfg(*entries):
        arr = (PerturbSpec * len(entries))(*[PerturbSpec(f.encode(), i, mode, amp, 0) for f, i, mode, amp in entries])
        return L.b2s_perturb_config(h, arr, len(entries))

    assert cfg(("dof_armature", -1, 1, 0.1)) == -1  # not declared
    assert cfg(("geom_solref", table, 0, 0.1)) == -1  # no slot for this geom
    assert cfg(("dof_damping", -1, 0, 1.0)) == -1  # scale amplitude >= 1
    assert cfg(("dof_damping", -1, 1, -0.1)) == -1  # negative amplitude
    assert cfg(("dof_damping", -1, 1, 2.0), ("geom_solimp", g, 0, 0.5)) == 0
    assert L.b2s_perturb_model(h, None, 1, 2 ** 32) == -1
    damp[1, 0] = -0.1
    solimp[2, 1] = float("nan")
    sim.set_const()
    assert sim.warn.cpu().tolist() == [0, 128, 128, 0]
    sim.close()
    # the friction-loss rows of every dof must fit the large tier
    small = BatchedSim(m, 2, precision="f32", maxefc=m.nv + 7)
    assert small._L.b2s_model_override(small._h, b"dof_frictionloss", -1) == -4
    small.close()
