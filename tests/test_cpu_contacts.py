"""CPU: the environment's contact queries (check_contact, get_contacts, _check_grasp, contact_geoms; robosuite_b200/envs/contacts.py)
on the oracle-backed stand-in with the contact export (tests/oracle_sim_export.py): geom resolution, the reference's matching
rules against the numpy restatement (tests/contact_ref.py), and the errors."""
import numpy as np
import pytest

from tests import contact_ref as ref
from tests.oracle_sim_export import ExportOracleSim

torch = pytest.importorskip("torch")


def _env(n=2, contact_queries=True, task="Lift"):
    import robosuite_b200 as suite

    return suite.make(task, robots="Panda", num_envs=n, seed=3, sim_cls=ExportOracleSim, precision="f64",
                      contact_queries=contact_queries)


@pytest.fixture(scope="module")
def env():
    e = _env()
    yield e
    e.close()


def _put(env, rows):
    """environment e's contact list := rows[e] (geom pairs by name); the rows after them are stale pairs that must be ignored"""
    gn = env.model.names["geom"]
    c = env.sim.contacts()
    c["geom"][:] = -1
    for e, pairs in enumerate(rows):
        c["ncon"][e] = len(pairs)
        for k, (a, b) in enumerate(pairs):
            c["geom"][e, k] = torch.tensor([gn.index(a), gn.index(b)], dtype=torch.int32)
        # a stale row beyond ncon: table-cube, which no query below may see
        c["geom"][e, len(pairs)] = torch.tensor([gn.index("table_collision"), gn.index("cube_g0")], dtype=torch.int32)


L_PAD, R_PAD = "gripper0_right_finger1_pad_collision", "gripper0_right_finger2_pad_collision"


def test_contact_geoms_by_prefix(env):
    m = env.model
    gn = m.names["geom"]
    colliding = {int(g) for p in m.pair_geom for g in p}
    grip = env.contact_geoms("gripper0_")
    assert gn.index(L_PAD) in grip and gn.index(R_PAD) in grip
    assert all(gn[g].startswith("gripper0_") and g in colliding for g in grip)
    robot = env.contact_geoms("robot0_")
    assert robot == sorted(g for g in colliding if gn[g].startswith("robot0_")) and len(robot) == 8
    assert env.contact_geoms("no_such_prefix") == []


def test_names_ids_and_tensors_resolve_alike(env):
    gn = env.model.names["geom"]
    _put(env, [[("table_collision", "cube_g0")], [(L_PAD, "cube_g0")]])
    cube, table = gn.index("cube_g0"), gn.index("table_collision")
    want = torch.tensor([True, False])
    for a, b in (("cube_g0", "table_collision"), (cube, table), ([cube], [table]), (torch.tensor([cube]), np.array([table])),
                 (["cube_g0"], [table, "floor"])):
        assert torch.equal(env.check_contact(a, b), want), (a, b)


def test_matching_rules(env):
    _put(env, [[("table_collision", "cube_g0"), (L_PAD, "floor")], [(L_PAD, "cube_g0"), (R_PAD, "cube_g0")]])
    t = lambda *x: torch.tensor(list(x))
    assert torch.equal(env.check_contact("cube_g0"), t(True, True))  # geoms_2 None: any partner, either side
    assert torch.equal(env.check_contact("table_collision"), t(True, False))
    assert torch.equal(env.check_contact("floor"), t(True, False))  # the second geom of the pair
    for a, b in (("cube_g0", "table_collision"), (L_PAD, "cube_g0"), ("floor", L_PAD), (R_PAD, "floor")):
        assert torch.equal(env.check_contact(a, b), env.check_contact(b, a)), (a, b)  # order symmetry
    assert torch.equal(env.check_contact(L_PAD, "cube_g0"), t(False, True))
    assert torch.equal(env.check_contact([L_PAD, R_PAD], ["floor", "cube_g0"]), t(True, True))
    assert torch.equal(env.check_contact(R_PAD, "floor"), t(False, False))
    gn = env.model.names["geom"]
    # get_contacts: the other geom of each contact with exactly one geom in the set; contacts inside the set are left out
    got = env.get_contacts(["cube_g0", "table_collision"])
    assert got.shape == (2, env.model.ngeom) and got.dtype == torch.bool
    assert torch.nonzero(got[0]).flatten().tolist() == []
    assert torch.nonzero(got[1]).flatten().tolist() == sorted([gn.index(L_PAD), gn.index(R_PAD)])
    assert torch.nonzero(env.get_contacts(L_PAD)[0]).flatten().tolist() == [gn.index("floor")]
    # _check_grasp: both fingerpad groups touch the object
    assert torch.equal(env._check_grasp("cube_g0"), t(False, True))
    assert torch.equal(env._check_grasp(["cube_g0"], gripper=[[L_PAD], R_PAD]), t(False, True))
    assert torch.equal(env._check_grasp("cube_g0", gripper=L_PAD), t(False, True))
    assert torch.equal(env._check_grasp("floor", gripper=L_PAD), t(True, False))


def test_queries_equal_the_restatement_after_steps():
    env = _env(n=3)
    m = env.model
    left, right = env._fingerpad_geoms()
    sets = [("cube_g0", None), ("cube_g0", "table_collision"), (env.contact_geoms("gripper0_"), "cube_g0"),
            (env.contact_geoms("robot0_"), None), ("table_collision", env.contact_geoms("gripper0_"))]
    rng = np.random.default_rng(0)
    act = np.zeros((3, 7))
    for t in range(4):
        act[:, :3] = [0, 0, -1]  # push down onto the cube / table
        act[:, 3:6] = rng.uniform(-0.2, 0.2, size=(3, 3))
        act[:, 6] = 1
        env.step(torch.as_tensor(act))
        c = env.sim.contacts()
        assert int(c["ncon"].min()) > 0
        for e in range(3):
            o = env.sim.o[e].contacts()
            assert c["geom"][e, : len(o)].tolist() == [[x["geom1"], x["geom2"]] for x in o]
            assert (c["geom"][e, len(o):] == -1).all()
        for a, b in sets:
            got = env.check_contact(a, b)
            assert got.tolist() == [ref.check_contact(m, c["ncon"][e], c["geom"][e], a, b) for e in range(3)], (t, a, b)
            g = env.get_contacts(a)
            for e in range(3):
                assert np.array_equal(g[e].numpy(), ref.get_contacts(m, c["ncon"][e], c["geom"][e], a)), (t, a)
        grasp = env._check_grasp(env.cube_geoms)
        assert grasp.tolist() == [ref.check_grasp(m, c["ncon"][e], c["geom"][e], [left, right], env.cube_geoms) for e in range(3)]
        assert grasp.tolist() == (env.sim.task_out[:, 2] > 0).tolist()
    env.close()


def test_errors():
    env = _env(contact_queries=False)
    for call in (lambda: env.check_contact("cube_g0"), lambda: env.get_contacts("cube_g0"), lambda: env._check_grasp("cube_g0")):
        with pytest.raises(RuntimeError, match="contact_queries=True"):
            call()
    env.close()
    env = _env()
    with pytest.raises(ValueError, match="unknown geom name 'no_such_geom'"):
        env.check_contact("no_such_geom")
    with pytest.raises(ValueError, match="unknown geom name"):
        env.check_contact("cube_g0", ["table_collision", "nope"])
    with pytest.raises(ValueError, match="out of range"):
        env.get_contacts(int(env.model.ngeom))
    with pytest.raises(ValueError, match="out of range"):
        env._check_grasp([-1])
    env.close()
