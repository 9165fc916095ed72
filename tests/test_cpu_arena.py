"""The tasks' arena arguments on the host: table_full_size / table_friction of Lift, Stack and NutAssembly (envs/base.py
table_model) and PickPlace's bin1_pos, bin2_pos, z_offset and z_rotation.  The recalled table rules are pinned against every
packaged model; the physics of a moved / thicker / rougher table runs on the fp64 oracle (no GPU)."""
import math

import numpy as np
import pytest
import torch
from scipy import stats

import robosuite_b200 as suite
from oracle.pyoracle import Oracle
from robosuite_b200.envs.base import table_model
from robosuite_b200.mjcf.compiler import GEOM_BOX, load_model, pack_model, primitive_geom_props
from tests.oracle_sim import OracleSim
from tests.oracle_sim_select import SelectOracleSim
from tests.util import ROOT

DEFAULT_SIZE, DEFAULT_FRICTION = (0.8, 0.8, 0.05), (1.0, 5e-3, 1e-4)
# (packaged model, table_offset, table_full_size) of every packaged model with a TableArena table
TABLE_MODELS = [("Lift_Panda", (0, 0, 0.8), DEFAULT_SIZE), ("Lift_Sawyer", (0, 0, 0.8), DEFAULT_SIZE),
                ("Stack_Panda", (0, 0, 0.8), DEFAULT_SIZE), ("Stack_Sawyer", (0, 0, 0.8), DEFAULT_SIZE),
                ("NutAssemblyRound_Panda", (0, 0, 0.82), DEFAULT_SIZE), ("Door_Panda", (-0.2, -0.35, 0.8), (0.8, 0.3, 0.05))]


def _pkg(name):
    return load_model("%s/robosuite_b200/assets/models/%s.npz" % (ROOT, name))


def _ids(m):
    return m.names["geom"].index("table_collision"), m.names["body"].index("table"), m.names["body"].index("robot0_base")


@pytest.mark.parametrize("name,offset,size", TABLE_MODELS)
def test_default_arguments_reproduce_every_packaged_table(name, offset, size):
    m = _pkg(name)
    t = table_model(m, offset, size, DEFAULT_FRICTION)
    g, tb, rb = _ids(m)
    for f, i in (("body_pos", tb), ("body_pos", rb), ("geom_size", g), ("geom_friction", g), ("geom_rbound", g), ("geom_aabb", g)):
        assert np.array_equal(getattr(t, f)[i], getattr(m, f)[i]), (name, f)
    # the model's own arrays are not touched
    assert t.body_pos is not m.body_pos and t.geom_size is not m.geom_size


@pytest.mark.parametrize("name,offset", [("Lift_Panda", (0, 0, 0.8)), ("Lift_Sawyer", (0, 0, 0.8)), ("NutAssemblyRound_Panda", (0, 0, 0.82))])
def test_non_default_batch_values(name, offset):
    m = _pkg(name)
    t = table_model(m, offset, (1.2, 0.6, 0.1), (2.0, 0.01, 2e-4))
    g, tb, rb = _ids(m)
    assert np.allclose(t.body_pos[tb], [0, 0, offset[2] - 0.05], rtol=0, atol=1e-15)
    assert np.allclose(t.body_pos[rb], [-0.16 - 0.6, m.body_pos[rb, 1], m.body_pos[rb, 2]], rtol=0, atol=1e-15)
    assert np.array_equal(t.geom_size[g], [0.6, 0.3, 0.05]) and np.array_equal(t.geom_friction[g], [2.0, 0.01, 2e-4])
    _, _, rb_, aabb = primitive_geom_props(GEOM_BOX, np.array([0.6, 0.3, 0.05]))
    assert t.geom_rbound[g] == rb_ and np.array_equal(t.geom_aabb[g], aabb)
    # translation of the robot changes none of the derived constants beyond rounding
    assert np.allclose(t.dof_invweight0, m.dof_invweight0, rtol=1e-9) and np.allclose(t.body_invweight0, m.body_invweight0, rtol=1e-9, atol=1e-12)


def _make(task="Lift", n=2, **kw):
    return suite.make(task, robots="Panda", num_envs=n, seed=0, sim_cls=OracleSim, precision="f64", **kw)


def test_env_edits_the_model_only_for_non_default_values():
    m = _pkg("Lift_Panda")
    b = _make(model=m, table_full_size=DEFAULT_SIZE, table_friction=list(DEFAULT_FRICTION))
    c = _make(model=m, table_full_size=(0.8, 0.8, 0.1))
    assert b.model is m  # defaults: the given model as is, no extra path
    assert c.model is not m and m.geom_size[_ids(m)[0], 2] == 0.025  # the caller's model is not written
    g, tb, rb = _ids(c.model)
    assert c.model.body_pos[tb, 2] == 0.8 - 0.05 and c.model.geom_size[g, 2] == 0.05


def _rest_height(thickness, steps=150):
    """z of a cube let go 1 mm above the top of a table of that thickness, after `steps` substeps of the oracle"""
    m = table_model(_pkg("Lift_Panda"), (0, 0, 0.8), (0.8, 0.8, thickness), DEFAULT_FRICTION)
    o = Oracle(pack_model(m))
    a = int(m.jnt_qposadr[m.names["joint"].index("cube_joint0")])
    h = float(m.geom_size[m.names["geom"].index("cube_g0"), 2])
    o.qpos[:] = m.qpos0
    o.qpos[a:a + 7] = [0.25, 0.25, 0.8 + h + 1e-3, 1, 0, 0, 0]
    for _ in range(steps):
        o.step()
    return float(o.qpos[a + 2]), h


def test_cube_rests_at_the_same_height_on_a_thick_table():
    z0, h = _rest_height(0.05)
    z1, _ = _rest_height(0.1)
    assert abs(z0 - (0.8 + h)) < 1e-3  # resting on the top (soft contact: a small penetration)
    assert abs(z1 - z0) < 1e-9


def _slide(friction, steps=60):
    """state of a cube resting on a table of that friction, pushed to 1 m/s along x, after `steps` substeps of the oracle"""
    m = table_model(_pkg("Lift_Panda"), (0, 0, 0.8), DEFAULT_SIZE, friction)
    o = Oracle(pack_model(m))
    j = m.names["joint"].index("cube_joint0")
    a, d = int(m.jnt_qposadr[j]), int(m.jnt_dofadr[j])
    h = float(m.geom_size[m.names["geom"].index("cube_g0"), 2])
    o.qpos[:] = m.qpos0
    o.qpos[a:a + 7] = [0.1, 0.25, 0.8 + h, 1, 0, 0, 0]
    for _ in range(100):
        o.step()
    o.qvel[d] = 1.0
    for _ in range(steps):
        o.step()
    return np.concatenate([o.qpos[a:a + 7], o.qvel[d:d + 6]])


def test_table_friction_mixes_by_maximum():
    """contact friction is the larger of the two geoms': a table smoother than the cube (1.0) changes no bit, a rougher one
    changes the slide"""
    base = _slide(DEFAULT_FRICTION)
    assert np.array_equal(_slide((0.5, 5e-3, 1e-4)), base)
    assert not np.allclose(_slide((2.0, 5e-3, 1e-4)), base, rtol=0, atol=1e-6)


@pytest.mark.parametrize("kw", [dict(table_full_size=(0.8, 0.8)), dict(table_full_size=(0.8, 0.8, 0.0)), dict(table_friction=(1, math.nan, 1)),
                                dict(table_friction=(-1, 0.1, 0.1)), dict(table_full_size=np.ones((3, 3))), dict(table_full_size=np.ones((2, 2)))])
def test_malformed_table_arguments_raise(kw):
    with pytest.raises(ValueError):
        _make(**kw)


def _pp(n=64, **kw):
    return suite.make("PickPlace", robots="Panda", num_envs=n, seed=3, sim_cls=SelectOracleSim, precision="f64", **kw)


def test_refusals():
    with pytest.raises(NotImplementedError, match="bins"):
        _pp(n=1, table_full_size=(0.8, 0.8, 0.05))
    with pytest.raises(NotImplementedError, match="bins"):
        _pp(n=1, table_friction=(2.0, 5e-3, 1e-4))
    with pytest.raises(NotImplementedError, match="Door"):
        suite.make("Door", num_envs=1, sim_cls=OracleSim, precision="f64", table_friction=(1.0, 5e-3, 1e-4))
    for kw in (dict(bin1_pos=(0, 0)), dict(bin2_pos=(0, math.inf, 0)), dict(z_offset=math.nan), dict(z_rotation=(0, 1, 2)),
               dict(z_rotation=math.inf)):
        with pytest.raises(ValueError):
            _pp(n=1, **kw)


def test_pick_place_defaults_change_nothing():
    m = _pkg("PickPlace_Panda")
    a, b = _pp(n=4), _pp(n=4, model=m, bin1_pos=(0.1, -0.25, 0.8), bin2_pos=[0.1, 0.28, 0.8], z_offset=0.0, table_full_size=(0.39, 0.49, 0.82))
    assert b.model is m
    assert torch.equal(a._reset_qpos, b._reset_qpos)


def test_pick_place_bins_placements_and_targets():
    b1, b2 = np.array([0.05, -0.3, 0.85]), np.array([0.15, 0.3, 0.78])
    env = _pp(bin1_pos=b1, bin2_pos=b2, z_offset=0.02, z_rotation=(0.2, 0.9))
    m = env.model
    for n, p in (("bin1", b1), ("bin2", b2)):
        assert np.array_equal(m.body_pos[m.names["body"].index(n)], p)
    ref = _pp()
    q, q0 = env._reset_qpos.numpy(), ref._reset_qpos.numpy()
    hx, hy = env.bin_size[0] / 2 - 0.05, env.bin_size[1] / 2 - 0.05
    yaws = []
    for name in env.obj_names:
        a = env.obj_qadr[name]
        assert np.all(np.abs(q[:, a] - b1[0]) <= hx) and np.all(np.abs(q[:, a + 1] - b1[1]) <= hy)
        assert np.allclose(q[:, a + 2] - q0[:, a + 2], 0.02 + b1[2] - 0.8, atol=1e-12)
        yaws.append(2 * np.arctan2(q[:, a + 6], q[:, a + 3]))
    assert stats.kstest(np.concatenate(yaws), stats.uniform(loc=0.2, scale=0.7).cdf).pvalue > 1e-3
    t = env.target_bin_placements
    assert np.allclose(t[:, 2], b2[2]) and np.allclose(t[:, :2].mean(0), b2[:2])
    xl, xh, yl, yh = env._bin_bounds(3)
    assert np.allclose([xl, xh, yl, yh], [b2[0], b2[0] + env.bin_size[0] / 2, b2[1], b2[1] + env.bin_size[1] / 2])


def test_pick_place_fixed_yaw():
    env = _pp(n=8, z_rotation=0.7)
    q = env._reset_qpos.numpy()
    for name in env.obj_names:
        a = env.obj_qadr[name]
        assert np.allclose(q[:, a + 3], math.cos(0.35), rtol=0, atol=1e-15) and np.allclose(q[:, a + 6], math.sin(0.35), rtol=0, atol=1e-15)


def test_domain_randomization_refuses_the_per_env_table_geom():
    from robosuite_b200.wrappers import BatchedDomainRandomizationWrapper
    from tests.oracle_sim_override import OverrideOracleSim

    env = suite.make("Lift", robots="Panda", num_envs=2, seed=0, sim_cls=OverrideOracleSim, precision="f64")
    env._table_ov = ()  # what per-environment table arguments set up (the CPU stand-in has no tree pose overrides)
    with pytest.raises(ValueError, match="table_collision"):
        BatchedDomainRandomizationWrapper(env, dynamics_randomization_args={"geom_names": ["table_collision"]})
