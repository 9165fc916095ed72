"""Host side of per-environment joint and contact fields and of dynamics randomisation: the host override model, the numpy
restatement of the device draws, and the host logic of BatchedDomainRandomizationWrapper on the CPU stand-in of the engine
(tests/oracle_sim_dynamics.py)."""
import numpy as np
import pytest
import torch

from robosuite_b200.mjcf import compiler
from tests.dynamics_override_host import dynamics_invalid, dynamics_override_model, perturb_values, philox4x32_10
from tests.util import load


def test_armature_changes_the_derived_constants_as_the_compiler_says():
    m = load("Lift_Panda")
    for f in (0.5, 3.0):
        arm = m.dof_armature * f + 0.01  # the cube's free joint has no armature in the model
        h = dynamics_override_model(m, dof_armature={-1: arm})
        # meaninertia is the mean diagonal of M: it moves by the mean change of the armature
        assert h.stat_meaninertia == pytest.approx(m.stat_meaninertia + np.mean(arm - m.dof_armature), rel=1e-12)
        ref = compiler.Model.__new__(compiler.Model)
        ref.__dict__.update({k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in m.__dict__.items()})
        ref.dof_armature = arm
        compiler._set_const(ref)
        for k in ("dof_invweight0", "body_invweight0"):
            assert np.array_equal(getattr(h, k), getattr(ref, k)), k
            assert not np.allclose(getattr(h, k), getattr(m, k)), k
        # more armature on every dof: every dof is harder to accelerate
        if f > 1:
            assert np.all(h.dof_invweight0 < m.dof_invweight0)
    assert np.array_equal(m.dof_armature, load("Lift_Panda").dof_armature)  # the input model is untouched


def test_contact_and_dof_fields_reach_the_host_model():
    m = load("Lift_Panda")
    g = m.names["geom"].index("cube_g0")
    h = dynamics_override_model(m, geom_solref={g: [0.03, 0.8]}, geom_solimp={g: [0.8, 0.9, 0.002, 0.5, 2]},
                                dof_damping={-1: m.dof_damping + 0.1}, dof_frictionloss={-1: np.full(m.nv, 0.05)})
    assert list(h.geom_solref[g]) == [0.03, 0.8] and list(h.geom_solimp[g]) == [0.8, 0.9, 0.002, 0.5, 2]
    assert np.array_equal(h.dof_damping, m.dof_damping + 0.1) and np.all(h.dof_frictionloss == 0.05)
    assert not dynamics_invalid(m, dof_damping={-1: m.dof_damping}, geom_solimp={g: m.geom_solimp[g]})
    assert dynamics_invalid(m, dof_damping={-1: np.r_[-1.0, m.dof_damping[1:]]})
    assert dynamics_invalid(m, dof_armature={-1: np.r_[np.inf, m.dof_armature[1:]]})
    assert dynamics_invalid(m, geom_solimp={g: [0.9, np.nan, 0.001, 0.5, 2]})
    assert dynamics_invalid(m, geom_solref={g: [np.inf, 1.0]})


def test_philox_known_answers():
    """the Random123 known-answer vectors of Philox4x32-10"""
    kat = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
           ((0xffffffff,) * 4, (0xffffffff, 0xffffffff), (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
           ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    for ctr, key, out in kat:
        assert tuple(int(x) for x in philox4x32_10(np.array(ctr, dtype=np.uint64), key)) == out


def test_perturbation_draws_bounds_and_independence():
    m = load("Lift_Panda")
    g, b = m.names["geom"].index("cube_g0"), m.names["body"].index("cube_main")
    spec = [("body_mass", b, "scale", 0.02), ("body_inertia", b, "scale", 0.02, True), ("geom_solimp", g, "scale", 0.1),
            ("dof_damping", None, "shift", 0.01), ("dof_frictionloss", 3, "shift", 0.05)]
    big = perturb_values(m, spec, range(64), seed=123, counter=7)
    small = perturb_values(m, spec, [0, 5, 63], seed=123, counter=7)
    for k in big:  # an environment's values depend only on (seed, counter, env, spec)
        assert np.array_equal(big[k][[0, 5, 63]], small[k])
    assert not np.array_equal(perturb_values(m, spec, [0], 123, 8)[0], big[0][:1])
    assert np.all(np.abs(big[0][:, 0] / m.body_mass[b] - 1) <= 0.02)
    ratio = big[1] / m.body_inertia[b]
    assert np.allclose(ratio, ratio[:, :1], rtol=1e-14) and np.all(np.abs(ratio - 1) <= 0.02)  # one draw for the three moments
    assert np.all(np.abs(big[2] / m.geom_solimp[g] - 1) <= 0.1)
    assert big[3].shape == (64, m.nv) and np.all(big[3] >= 0) and np.all(big[3] <= m.dof_damping + 0.01)
    assert (big[3][:, m.dof_damping == 0] == 0).any()  # shift mode is clipped at 0
    assert big[4].shape == (64, 1) and np.all(big[4] <= m.dof_frictionloss[3] + 0.05)


def _make(task, n=2, sim=True, **kw):
    import robosuite_b200 as suite
    from tests.oracle_sim_dynamics import DynamicsOracleSim

    return suite.make(task, robots="Panda", num_envs=n, seed=0, sim_cls=DynamicsOracleSim if sim else None, **kw)


@pytest.mark.parametrize("task,ngeom,bodies", [("Lift", 3, ["cube_main"]), ("Stack", 4, ["cubeA_main", "cubeB_main"]),
                                               ("Door", 7, ["Door_door", "Door_latch"]),
                                               ("PickPlace", 2, ["Milk_main", "Bread_main", "Cereal_main", "Can_main"])])
def test_default_selection_on_the_packaged_tasks(task, ngeom, bodies):
    from robosuite_b200.wrappers import BatchedDomainRandomizationWrapper

    env = _make(task)
    w = BatchedDomainRandomizationWrapper(env, seed=1)
    m = env.model
    assert [m.names["body"][b] for b in w.default_bodies()] == bodies
    geoms = sorted({i for f, i, *_ in w.perturb_spec if f.startswith("geom_")})
    assert len(geoms) == ngeom
    left, right = env._fingerpad_geoms()
    assert set(left + right) <= set(geoms)
    fields = {f for f, *_ in w.perturb_spec}
    assert fields == {"body_mass", "body_inertia", "geom_friction", "geom_solref", "geom_solimp", "dof_damping", "dof_armature",
                      "dof_frictionloss"}
    assert {(f, i) for f, i, *_ in w.perturb_spec if f.startswith("dof_")} == {(f, -1) for f in ("dof_damping", "dof_armature", "dof_frictionloss")}
    # every selected object has its per-environment array
    for f, i, *_ in w.perturb_spec:
        assert env.sim.model_override(f, None if f.startswith("dof_") else i).shape[0] == env.num_envs


def test_nut_assembly_needs_explicit_geoms():
    from robosuite_b200.wrappers import BatchedDomainRandomizationWrapper

    env = _make("NutAssemblyRound")
    with pytest.raises(NotImplementedError, match="geom_names"):
        BatchedDomainRandomizationWrapper(env)
    w = BatchedDomainRandomizationWrapper(env, dynamics_randomization_args={"geom_names": ["SquareNut_g0", "RoundNut_g0"]})
    assert sorted({i for f, i, *_ in w.perturb_spec if f.startswith("geom_")}) == sorted(
        env.model.names["geom"].index(n) for n in ("SquareNut_g0", "RoundNut_g0"))


def test_knobs_the_engine_cannot_honour():
    from robosuite_b200.wrappers import BatchedDomainRandomizationWrapper

    env = _make("Lift")
    for knob in ("randomize_position", "randomize_quaternion", "randomize_stiffness", "randomize_density", "randomize_viscosity"):
        with pytest.raises(NotImplementedError, match=knob):
            BatchedDomainRandomizationWrapper(env, dynamics_randomization_args={knob: True})
    for knob in ("randomize_color", "randomize_camera", "randomize_lighting"):
        with pytest.raises(NotImplementedError, match=knob):
            BatchedDomainRandomizationWrapper(env, **{knob: True})
    with pytest.raises(ValueError, match="unknown"):
        BatchedDomainRandomizationWrapper(env, dynamics_randomization_args={"randomize_mas": True})
    with pytest.raises(ValueError, match="unknown body"):
        BatchedDomainRandomizationWrapper(env, dynamics_randomization_args={"body_names": ["no_such_body"]})
    cube = _make("Lift", per_env_cube_size=True)
    with pytest.raises(ValueError, match="per_env_cube_size"):
        BatchedDomainRandomizationWrapper(cube)
    # the task's own cube draws and the wrapper's friction / contact draws coexist
    w = BatchedDomainRandomizationWrapper(cube, dynamics_randomization_args={"randomize_mass": False, "randomize_inertia": False})
    assert not any(f.startswith("body_") for f, *_ in w.perturb_spec)


def test_explicit_joints_select_their_dofs():
    from robosuite_b200.wrappers import BatchedDomainRandomizationWrapper

    env = _make("Lift")
    m = env.model
    w = BatchedDomainRandomizationWrapper(env, dynamics_randomization_args={"joint_names": ["robot0_joint2", "cube_joint0"],
                                                                            "randomize_armature": False, "randomize_frictionloss": False})
    j2, cj = m.names["joint"].index("robot0_joint2"), m.names["joint"].index("cube_joint0")
    want = [int(m.jnt_dofadr[j2])] + list(range(int(m.jnt_dofadr[cj]), int(m.jnt_dofadr[cj]) + 6))
    assert [i for f, i, *_ in w.perturb_spec if f == "dof_damping"] == want
    assert not any(f in ("dof_armature", "dof_frictionloss") for f, *_ in w.perturb_spec)


def test_wrapper_masks_follow_the_episode_clocks():
    """per-environment `timestep % n == 0` masks before each step, the counter advancing per call, and the perturbed environments'
    override arrays changing while the others stay"""
    from robosuite_b200.wrappers import BatchedDomainRandomizationWrapper

    n, k = 4, 3
    env = _make("Lift", n=n)
    w = BatchedDomainRandomizationWrapper(env, seed=9, randomize_every_n_steps=k)
    env.set_episode_steps([0, 1, 2, 4])
    sim = env.sim
    zero = torch.zeros((n, env.action_dim), dtype=torch.float64)
    damp = sim.model_override("dof_damping")
    for step in range(4):
        clocks = env.timestep.clone()
        before = damp.clone()
        w.step(zero)
        mask, seed, counter = sim.perturb_calls[-1]
        due = (clocks % k == 0)
        assert torch.equal(mask.bool(), due) and seed == 9 and counter == step
        assert torch.equal(damp[~due], before[~due])
        ref = perturb_values(env.model, sim._pert, [e for e in range(n) if due[e]], 9, counter)
        kd = [f for f, *_ in sim._pert].index("dof_damping")
        assert np.array_equal(damp[due].numpy(), ref[kd])
    assert w.counter == 4


def test_gym_auto_reset_randomizes_exactly_the_finished_environments():
    from robosuite_b200.wrappers import BatchedDomainRandomizationWrapper, BatchedGymWrapper

    n = 4
    env = _make("Lift", n=n, horizon=3)
    w = BatchedDomainRandomizationWrapper(env, seed=2, randomize_every_n_steps=0)
    g = BatchedGymWrapper(w)
    g.reset()
    assert env.sim.perturb_calls[-1][0] is None  # a full reset randomises every environment
    env.set_episode_steps([0, 1, 2, 2])
    mass = env.sim.model_override("body_mass", env.cube_body_id)
    ncalls = len(env.sim.perturb_calls)
    m0 = mass.clone()
    g.step(np.zeros((n, env.action_dim)))
    mask = env.sim.perturb_calls[-1][0]
    assert len(env.sim.perturb_calls) == ncalls + 1
    assert mask.bool().tolist() == [False, False, True, True]
    assert torch.equal(mass[:2], m0[:2]) and bool((mass[2:] != m0[2:]).all())
    assert env.timestep.tolist() == [1, 2, 0, 0]


@pytest.mark.skipif(not __import__("os").environ.get("ROBOSUITE_REFERENCE"), reason="needs a reference robosuite checkout: set ROBOSUITE_REFERENCE")
def test_default_magnitudes_match_the_reference():
    """the perturbation magnitudes of DEFAULT_DYNAMICS_ARGS, read from the reference's source without importing it"""
    import ast
    import os

    from robosuite_b200.wrappers import DEFAULT_DYNAMICS_ARGS

    src = open(os.path.join(os.environ["ROBOSUITE_REFERENCE"], "robosuite", "wrappers", "domain_randomization_wrapper.py")).read()
    node = next(n for n in ast.walk(ast.parse(src)) if isinstance(n, ast.Assign) and getattr(n.targets[0], "id", "") == "DEFAULT_DYNAMICS_ARGS")
    ref = ast.literal_eval(node.value)
    for k, v in DEFAULT_DYNAMICS_ARGS.items():
        if k.endswith(("_ratio", "_size")):
            assert ref[k] == v, k
