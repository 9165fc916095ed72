"""Host side of per-environment model values: the factored per-type geom rules, the host override model the oracles are built from,
and BatchedLift(per_env_cube_size=True) on the CPU stand-in of the engine (tests/oracle_sim_override.py)."""
import glob
import os

import numpy as np
import pytest
import torch

from robosuite_b200.mjcf import compiler
from tests.model_override_host import invalid, override_model
from tests.util import ROOT, load

PACKAGED = sorted(glob.glob(os.path.join(ROOT, "robosuite_b200", "assets", "models", "*.npz")))


@pytest.mark.parametrize("path", PACKAGED, ids=[os.path.basename(p)[:-4] for p in PACKAGED])
def test_override_model_without_values_reproduces_the_compiled_constants(path):
    m = compiler.load_model(path)
    h = override_model(m, geom_size={g: m.geom_size[g] for g in range(m.ngeom) if int(m.geom_type[g]) in (2, 3, 4, 5, 6)})
    for k in ("geom_rbound", "geom_aabb", "body_invweight0", "dof_invweight0"):
        assert np.array_equal(getattr(h, k), getattr(m, k)), k
    assert h.stat_meaninertia == m.stat_meaninertia


def test_override_model_recomputes_bounds_and_constants():
    m = load("Lift_Panda")
    g, b = m.names["geom"].index("cube_g0"), m.names["body"].index("cube_main")
    h = override_model(m, geom_size={g: [0.05, 0.04, 0.03]}, body_mass={b: 3 * m.body_mass[b]})
    assert h.geom_rbound[g] == pytest.approx(np.sqrt(0.05 ** 2 + 0.04 ** 2 + 0.03 ** 2))
    assert list(h.geom_aabb[g]) == [0, 0, 0, 0.05, 0.04, 0.03]
    # a heavier cube is harder to push: its translational inverse weight drops by the mass ratio
    assert h.body_invweight0[b, 0] == pytest.approx(m.body_invweight0[b, 0] / 3, rel=1e-9)
    assert np.array_equal(m.geom_size[g], load("Lift_Panda").geom_size[g])  # the input model is untouched


def test_primitive_geom_props_rules():
    P = compiler.primitive_geom_props
    assert P(compiler.GEOM_SPHERE, np.array([0.1, 0, 0]))[2:] == (0.1, [0, 0, 0, 0.1, 0.1, 0.1])
    assert P(compiler.GEOM_CAPSULE, np.array([0.1, 0.2, 0]))[2] == pytest.approx(0.3)
    assert P(compiler.GEOM_CYLINDER, np.array([0.3, 0.4, 0]))[2] == pytest.approx(0.5)
    assert P(compiler.GEOM_ELLIPSOID, np.array([0.1, 0.3, 0.2]))[2] == pytest.approx(0.3)
    assert P(compiler.GEOM_PLANE, np.zeros(3))[3] == [0, 0, -1e10, 1e10, 1e10, 1e10]


def test_invalid_override_values():
    m = load("Lift_Panda")
    g, b = m.names["geom"].index("cube_g0"), m.names["body"].index("cube_main")
    assert not invalid(m, geom_size={g: m.geom_size[g]}, body_mass={b: m.body_mass[b]}, body_inertia={b: m.body_inertia[b]})
    assert invalid(m, geom_size={g: [0.02, 0.0, 0.02]})
    assert invalid(m, geom_friction={g: [1.0, np.inf, 1e-4]})
    assert invalid(m, body_mass={b: -1.0})
    assert invalid(m, body_inertia={b: [1e-5, 1e-5, 3e-5]})


def _lift(n, seed=0, **kw):
    import robosuite_b200 as suite
    from tests.oracle_sim_override import OverrideOracleSim

    return suite.make("Lift", robots="Panda", num_envs=n, seed=seed, sim_cls=OverrideOracleSim, **kw)


def test_lift_per_env_cube_size_on_the_oracle():
    n = 4
    env = _lift(n, per_env_cube_size=True, hard_reset=True)
    m = env.model
    g, b = m.names["geom"].index("cube_g0"), env.cube_body_id
    size, mass, inertia = (t.numpy().copy() for t in env._cube_ov)
    assert size.min() >= 0.020 and size.max() <= 0.022 and len(np.unique(size[:, 0])) == n
    W = (compiler.quat2mat(m.body_iquat[b]).T @ compiler.quat2mat(m.geom_quat[g])) ** 2
    for e in range(n):
        s = size[e]
        assert mass[e] == pytest.approx(8000 * np.prod(s), rel=1e-12)
        box = mass[e] / 3 * np.array([s[1] ** 2 + s[2] ** 2, s[0] ** 2 + s[2] ** 2, s[0] ** 2 + s[1] ** 2])
        assert np.allclose(inertia[e], W @ box, rtol=1e-12)
        # each oracle runs the environment's own cube
        o = env.sim.o[e]
        assert o.ncon >= 0
    # the model's own cube under the box rule in the inertial frame gives the compiled fixture's moments
    s = m.geom_size[g]
    box = m.body_mass[b] / 3 * np.array([s[1] ** 2 + s[2] ** 2, s[0] ** 2 + s[2] ** 2, s[0] ** 2 + s[1] ** 2])
    assert np.allclose(W @ box, m.body_inertia[b], rtol=1e-6)
    assert np.allclose(env.sim.qpos[:, env.cube_qadr + 2].numpy(), 0.81 + size[:, 2])
    zero = torch.zeros((n, env.action_dim), dtype=torch.float64)
    for _ in range(3):
        env.step(zero)
    mask = torch.tensor([True, False, True, False])
    env.reset(mask=mask)
    s1 = env._cube_ov[0].numpy()
    assert np.array_equal(s1[~mask.numpy()], size[~mask.numpy()]) and not np.any(s1[mask.numpy()] == size[mask.numpy()])
    assert int(env.sim.warn.abs().max()) == 0
    env.sim.model_override("body_mass", b)[1] = -1.0
    env.sim.set_const(torch.tensor([0, 1, 0, 0], dtype=torch.uint8))
    assert env.sim.warn.tolist() == [0, 128, 0, 0]


def test_lift_cube_size_draws_only_when_asked():
    a, b = _lift(2, seed=3), _lift(2, seed=3, per_env_cube_size=False)
    assert torch.equal(a._reset_qpos, b._reset_qpos) and a._cube_ov is None
    c = _lift(2, seed=3, per_env_cube_size=True)  # hard_reset=False: drawn once
    # the robot's and the cube placement's draws come first: everything but the cube height is where it is without the option
    assert torch.equal(a._reset_qpos[:, :11], c._reset_qpos[:, :11])
    s0 = c._cube_ov[0].clone()
    c.reset()
    assert torch.equal(c._cube_ov[0], s0)
