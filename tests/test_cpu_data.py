"""CPU: the batched MjData view (BatchedSim.data, robosuite_b200/data.py) on the oracle-backed stand-in with the step-1 export
(tests/oracle_sim_export.py): name and id resolution, shapes, the xmat reshapes, the point velocities restated in numpy, and the
errors."""
import numpy as np
import pytest

from tests.oracle_sim_export import ExportOracleSim

torch = pytest.importorskip("torch")

SITE, BODY, GEOM = "gripper0_right_grip_site", "cube_main", "cube_g0"


def _env(n=2, data_queries=True, task="Lift"):
    import robosuite_b200 as suite

    return suite.make(task, robots="Panda", num_envs=n, seed=3, sim_cls=ExportOracleSim, precision="f64", data_queries=data_queries)


@pytest.fixture(scope="module")
def env():
    e = _env()
    rng = np.random.default_rng(0)
    for _ in range(2):
        e.step(torch.as_tensor(rng.uniform(-1, 1, size=(2, e.action_dim))))
    yield e
    e.close()


def test_make_switches_the_export_on(env):
    assert env.sim.step1_export and not env.sim.full_export


def test_shapes_and_resolution(env):
    m, d = env.model, env.sim.data
    nb, ns, ng, nv = m.nbody, m.nsite, m.ngeom, m.nv
    shapes = {"body_xpos": (2, nb, 3), "body_xquat": (2, nb, 4), "body_xmat": (2, nb, 9), "site_xpos": (2, ns, 3),
              "site_xmat": (2, ns, 9), "geom_xpos": (2, ng, 3), "geom_xmat": (2, ng, 9), "qM": (2, nv, nv), "cdof": (2, nv, 6),
              "qfrc_bias": (2, nv), "qfrc_passive": (2, nv)}
    for k, s in shapes.items():
        assert tuple(getattr(d, k).shape) == s, k
    assert tuple(d.full_m().shape) == (2, nv, nv) and torch.equal(d.full_m(), d.qM)
    ids = {"body": m.names["body"].index(BODY), "site": m.names["site"].index(SITE), "geom": m.names["geom"].index(GEOM)}
    names = {"body": BODY, "site": SITE, "geom": GEOM}
    for kind, i in ids.items():
        pos = {"body": d.body_xpos, "site": d.site_xpos, "geom": d.geom_xpos}[kind][:, i]
        for key in (names[kind], i, np.int64(i)):
            assert torch.equal(getattr(d, "get_%s_xpos" % kind)(key), pos), (kind, key)
            for f in ("jacp", "jacr"):
                j = getattr(d, "get_%s_%s" % (kind, f))(key)
                assert tuple(j.shape) == (2, 3, nv), (kind, f)
            for f in ("xvelp", "xvelr"):
                assert tuple(getattr(d, "get_%s_%s" % (kind, f))(key).shape) == (2, 3), (kind, f)
    assert torch.equal(d.get_body_xquat(BODY), d.body_xquat[:, ids["body"]])
    # the rows are the oracle's own arrays of the last substep's step1
    for e in range(2):
        o = env.sim.o[e]
        assert np.array_equal(d.get_body_xpos(BODY)[e].numpy(), o.xpos[ids["body"]])
        assert np.array_equal(d.get_site_xpos(SITE)[e].numpy(), o.site_xpos[ids["site"]])
        assert np.array_equal(d.qM[e].numpy(), o.M)
    # the cube's position is what the task's observation reads
    assert torch.equal(d.get_body_xpos(BODY), env.sim.xpos[:, env.cube_body_id])


def test_xmat_reshapes(env):
    m, d = env.model, env.sim.data
    for kind, name, flat in (("body", BODY, d.body_xmat), ("site", SITE, d.site_xmat), ("geom", GEOM, d.geom_xmat)):
        i = m.names[kind].index(name)
        got = getattr(d, "get_%s_xmat" % kind)(name)
        assert tuple(got.shape) == (2, 3, 3)
        for e in range(2):
            assert np.array_equal(got[e].numpy(), flat[e, i].numpy().reshape(3, 3)), kind
            # a rotation: orthonormal with determinant 1
            assert np.allclose(got[e].numpy() @ got[e].numpy().T, np.eye(3), atol=1e-12), kind


def test_velocities_are_jacobian_times_qvel(env):
    d = env.sim.data
    qvel = env.sim.qvel.numpy()
    assert np.abs(qvel).max() > 1e-3  # the arm is moving
    for kind, name in (("body", BODY), ("site", SITE), ("geom", GEOM), ("body", "robot0_right_hand")):
        for f, jf in (("xvelp", "jacp"), ("xvelr", "jacr")):
            v = getattr(d, "get_%s_%s" % (kind, f))(name).numpy()
            J = getattr(d, "get_%s_%s" % (kind, jf))(name).numpy()
            for e in range(2):
                assert np.allclose(v[e], np.dot(J[e], qvel[e]), rtol=0, atol=1e-12), (kind, name, f)
    # the site Jacobian of the hand's grip site moves with the arm's dofs only
    jp = d.get_site_jacp(SITE).numpy()
    arm = env._ref_joint_vel_indexes
    assert np.abs(jp[:, :, arm]).max() > 0
    other = [i for i in range(env.model.nv) if i not in arm]
    assert np.abs(jp[:, :, other]).max() == 0


def test_errors():
    env = _env(data_queries=False)
    d = env.sim.data
    calls = (lambda: d.body_xpos, lambda: d.qM, lambda: d.full_m(), lambda: d.get_site_xpos(SITE),
             lambda: d.get_body_jacp(BODY), lambda: d.get_geom_xvelr(GEOM), lambda: d.qfrc_bias)
    for call in calls:
        with pytest.raises(RuntimeError, match=r"data_queries=True.*set_step1_export"):
            call()
    env.sim.set_step1_export(True)
    assert tuple(d.get_site_xpos(SITE).shape) == (2, 3)
    env.sim.set_step1_export(False)
    env.sim.set_export(True)  # the full export also writes the arrays
    assert tuple(d.get_site_xpos(SITE).shape) == (2, 3)
    m = env.model
    with pytest.raises(ValueError, match="No \"site\" with name 'no_such_site'"):
        d.get_site_xpos("no_such_site")
    with pytest.raises(ValueError, match="body id .* out of range"):
        d.get_body_jacp(m.nbody)
    with pytest.raises(ValueError, match="out of range"):
        d.get_site_xmat(-1)
    colliding = {int(g) for p in m.pair_geom for g in p}
    visual = next(g for g in range(m.ngeom) if g not in colliding)
    for key in (visual, m.names["geom"][visual]):
        for call in (d.get_geom_xpos, d.get_geom_xmat, d.get_geom_jacp, d.get_geom_xvelp):
            with pytest.raises(ValueError, match="non-colliding"):
                call(key)
    env.close()
