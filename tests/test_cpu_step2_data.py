"""CPU: the step-2 half of the batched MjData view (BatchedSim.data's forces, constraint rows and contact_force(),
robosuite_b200/data.py) on the oracle-backed stand-in with the step-2 export and the contact records
(tests/oracle_sim_export.py): make(..., dynamics_queries=True), shapes, contact_force() against the oracle's rows contact by
contact, the resting cube's contact forces summing to its weight, and the errors."""
import copy
import types

import numpy as np
import pytest

from tests.oracle_sim_export import ExportOracleSim

torch = pytest.importorskip("torch")

N = 2


def _env(dynamics_queries=True, **kw):
    import robosuite_b200 as suite

    return suite.make("Lift", robots="Panda", num_envs=N, seed=3, sim_cls=ExportOracleSim, precision="f64",
                      dynamics_queries=dynamics_queries, **kw)


@pytest.fixture(scope="module")
def env():
    """Lift after the cube has settled on the table under zero actions (the arm holds its pose above it)"""
    e = _env()
    for _ in range(8):
        e.step(torch.zeros((N, e.action_dim), dtype=torch.float64))
    yield e
    e.close()


def test_make_switches_both_exports_on(env):
    s = env.sim
    assert s.step2_export and s.contact_export and not s.full_export and not s.step1_export
    plain = _env(dynamics_queries=False)
    assert not plain.sim.step2_export and not plain.sim.contact_export
    plain.close()


def test_shapes(env):
    m, d = env.model, env.sim.data
    nv, nu = m.nv, m.nu
    me, mc = env.sim.efc_force.shape[1], env.sim.contact_efc_address.shape[1]
    shapes = {"qacc": (N, nv), "qfrc_actuator": (N, nv), "actuator_force": (N, nu), "qfrc_smooth": (N, nv),
              "qacc_smooth": (N, nv), "qfrc_constraint": (N, nv), "nefc": (N,), "efc_type": (N, me), "efc_J": (N, me, nv),
              "efc_D": (N, me), "efc_R": (N, me), "efc_aref": (N, me), "efc_force": (N, me), "solver_niter": (N,)}
    for k, s in shapes.items():
        assert tuple(getattr(d, k).shape) == s, k
    assert tuple(d.contact_force().shape) == (N, mc, 6)
    assert tuple(d.contact_force(0).shape) == (N, 6)
    # the views are the oracle's own arrays of the last substep
    for e in range(N):
        o = env.sim.o[e]
        n = int(d.nefc[e])
        assert n == o.nefc and n > 0
        assert np.array_equal(d.qfrc_constraint[e].numpy(), o.qfrc_constraint)
        assert np.array_equal(d.actuator_force[e].numpy(), o.actuator_force)
        assert np.array_equal(d.efc_force[e, :n].numpy(), o.efc("force"))
        assert np.array_equal(d.efc_J[e, :n].numpy(), o.efc("J"))
        assert not d.efc_force[e, n:].any() and not d.efc_D[e, n:].any()
        assert np.array_equal(d.qacc[e].numpy(), o.qacc)


def test_contact_force_is_the_rows_of_each_contact(env):
    d = env.sim.data
    f = d.contact_force().numpy()
    mc = f.shape[1]
    seen_rows = seen_none = 0
    for e in range(N):
        o = env.sim.o[e]
        cons = o.contacts()
        assert int(env.sim.ncon[e]) == len(cons)
        rows = o.efc("force")
        for c in range(mc):
            want = np.zeros(6)
            if c < len(cons) and cons[c]["efc_address"] >= 0:
                a, dim = cons[c]["efc_address"], cons[c]["dim"]
                want[:dim] = rows[a:a + dim]
                seen_rows += 1
            elif c < len(cons):
                seen_none += 1
            assert np.array_equal(f[e, c], want), (e, c)
            assert np.array_equal(d.contact_force(c)[e].numpy(), want), (e, c)
        assert not f[e, len(cons):].any()
    assert seen_rows > 0  # the cube rests on the table


def test_resting_cube_contact_forces_sum_to_its_weight(env):
    m, s = env.model, env.sim
    f = s.data.contact_force().numpy()
    frame = s.contact_frame.numpy().reshape(N, -1, 3, 3)
    geom = s.contact_geom.numpy()
    body = np.asarray(m.geom_bodyid)
    b = env.cube_body_id
    g = -float(np.asarray(m.opt_gravity)[2])
    weight = float(np.asarray(m.body_mass)[b]) * g
    for e in range(N):
        total = np.zeros(3)
        for c in range(int(s.ncon[e])):
            g1, g2 = geom[e, c]
            if b not in (body[g1], body[g2]):
                continue
            world = frame[e, c].T @ f[e, c, :3]  # the force geom1 exerts on geom2, along the normal from geom1 to geom2
            total += world if body[g2] == b else -world
        assert abs(total[2] - weight) < 1e-3 * weight, (e, total, weight)
        assert np.abs(total[:2]).max() < 1e-3 * weight, (e, total)


def test_errors():
    env = _env(dynamics_queries=False)
    d = env.sim.data
    assert tuple(d.qacc.shape) == (N, env.model.nv)  # state: no export needed
    calls = (lambda: d.qfrc_actuator, lambda: d.actuator_force, lambda: d.efc_force, lambda: d.efc_J, lambda: d.nefc,
             lambda: d.solver_niter, lambda: d.qfrc_constraint, lambda: d.contact_force())
    for call in calls:
        with pytest.raises(RuntimeError, match=r"dynamics_queries=True.*set_step2_export"):
            call()
    env.sim.set_step2_export(True)
    assert tuple(d.efc_force.shape)[0] == N
    with pytest.raises(RuntimeError, match=r"contact records.*set_contact_export"):
        d.contact_force()
    env.sim.set_contact_export(True)
    assert tuple(d.contact_force(1).shape) == (N, 6)
    with pytest.raises(ValueError, match="out of range"):
        d.contact_force(env.sim.contact_efc_address.shape[1])
    env.sim.set_step2_export(False)
    env.sim.set_contact_export(False)
    env.sim.set_export(True)  # the full export writes both
    assert tuple(d.contact_force().shape)[0] == N and tuple(d.efc_D.shape)[0] == N
    # the step-1 check keeps its own message
    env.sim.set_export(False)
    with pytest.raises(RuntimeError, match=r"data_queries=True.*set_step1_export"):
        d.body_xpos
    # pyramidal cones: not a wrong answer
    from robosuite_b200.data import BatchedData

    pm = copy.copy(env.model)
    pm.opt_cone = 0
    sim = types.SimpleNamespace(model=pm, full_export=True, step2_export=True, contact_export=True)
    with pytest.raises(NotImplementedError, match="elliptic"):
        BatchedData(sim).contact_force()
    env.close()


def test_contact_force_never_reads_past_the_rows():
    """contact records and rows from different steps (the contact export switched on after the step-2 export's last write): a
    stale dim or address must not index past nefc or past efc_force's capacity"""
    env = _env()
    env.step(torch.zeros((N, env.action_dim), dtype=torch.float64))
    s = env.sim
    me = s.efc_force.shape[1]
    s.ncon[:] = torch.clamp(s.ncon, min=2)
    s.contact_dim[:, 0], s.contact_efc_address[:, 0] = 6, me - 2     # would reach past the capacity
    s.contact_dim[:, 1], s.contact_efc_address[:, 1] = 6, s.nefc - 1  # would reach past the solve's rows
    f = s.data.contact_force().numpy()
    for e in range(N):
        n = int(s.nefc[e])
        assert not f[e, 0].any() or n > me - 2
        rows = s.efc_force[e].numpy()
        assert np.array_equal(f[e, 1], np.concatenate([rows[n - 1:n], np.zeros(5)]))
    env.close()
