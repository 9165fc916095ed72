"""Object placement samplers (robosuite_b200/placement_samplers.py): the class API and its defaults, the lowering of every option
into the device program, the numpy restatement of b2s_place_objects (tests/placement_ref.py) against a transcription of the
reference's sample() loop fed the same uniforms, every host-side error, and every task placing its objects through the host layer on
the CPU stand-in (tests/oracle_sim_placement.py)."""
import math

import numpy as np
import pytest
import torch

import robosuite_b200 as suite
from robosuite_b200.envs.base import SIM_WARN_BITS
from robosuite_b200.errors import RandomizationError
from robosuite_b200.placement_samplers import (ObjectPositionSampler, SequentialCompositeSampler, UniformRandomSampler,
                                               lower)
from tests.oracle_sim_placement import PlacementOracleSim
from tests.placement_ref import PhiloxStream, place_env, place_values, reference_sample, sincos

OBJ = {"a": dict(radius=0.03, bottom=-0.02, top=0.02, qpos_adr=9, body=-1),
       "b": dict(radius=0.04, bottom=-0.025, top=0.025, qpos_adr=16, body=-1),
       "c": dict(radius=0.05, bottom=-0.05, top=0.05, qpos_adr=23, body=-1)}


def test_class_api_and_defaults():
    s = UniformRandomSampler("S")
    assert (s.name, s.mujoco_objects, s.x_range, s.y_range, s.rotation, s.rotation_axis) == ("S", [], (0, 0), (0, 0), None, "z")
    assert s.ensure_object_boundary_in_range and s.ensure_valid_placement
    assert s.reference_pos == (0, 0, 0) and s.z_offset == 0.0
    s.add_objects("a")
    s.add_objects(["b"])
    assert s.mujoco_objects == ["a", "b"]
    s.reset()
    assert s.mujoco_objects == []
    with pytest.raises(NotImplementedError):
        s.sample()
    c = SequentialCompositeSampler("C")
    assert isinstance(c, ObjectPositionSampler) and list(c.samplers) == [] and c.mujoco_objects == []
    c.append_sampler(UniformRandomSampler("A", mujoco_objects="a"), sample_args={"on_top": False})
    c.hide("b")
    assert list(c.samplers) == ["A", "HideSampler"] and c.mujoco_objects == ["a", "b"]
    h = c.samplers["HideSampler"]
    assert (h.x_range, h.y_range, h.rotation, h.rotation_axis, h.z_offset) == ((-10, -20), (-10, -20), [0, 0], "z", 10)
    assert not h.ensure_object_boundary_in_range and not h.ensure_valid_placement
    c.add_objects_to_sampler("A", "c")
    assert c.samplers["A"].mujoco_objects == ["a", "c"] and "c" in c.mujoco_objects
    c.reset()
    assert c.mujoco_objects == [] and all(not x.mujoco_objects for x in c.samplers.values())


@pytest.mark.parametrize("kw", [dict(x_range=(0, math.inf)), dict(y_range=(math.nan, 0)), dict(x_range=(0,)), dict(z_offset=math.nan),
                                dict(reference_pos=(0, 0, math.inf)), dict(reference_pos=(0, 0)), dict(rotation=math.nan),
                                dict(rotation=(0, math.inf)), dict(rotation=[(0, 1)] * 9), dict(rotation_axis="w"),
                                dict(rotation_axis="Z")])
def test_constructor_rejects_bad_values(kw):
    with pytest.raises(ValueError):
        UniformRandomSampler("S", **kw)


def test_composite_errors():
    c = SequentialCompositeSampler("C")
    c.append_sampler(UniformRandomSampler("A", mujoco_objects="a"))
    with pytest.raises(ValueError):
        c.append_sampler(UniformRandomSampler("B", mujoco_objects="a"))  # already has a sampler
    with pytest.raises(ValueError):
        c.append_sampler(UniformRandomSampler("B", mujoco_objects="b"), sample_args={"fixtures": None})
    with pytest.raises(ValueError):
        c.append_sampler(UniformRandomSampler("B", mujoco_objects="b"), sample_args={"reference": (0, math.nan, 0)})
    with pytest.raises(ValueError):
        UniformRandomSampler("A", mujoco_objects="a").add_objects("a")


def _one(**kw):
    return lower(UniformRandomSampler("S", mujoco_objects=["a"], **kw), {"a": OBJ["a"]})[1][0]


def test_lowering_ranges_boundary_and_validity():
    e = _one(x_range=(0.2, -0.1), y_range=(-0.3, 0.4), ensure_object_boundary_in_range=False, ensure_valid_placement=False)
    assert (e["x_min"], e["x_max"], e["y_min"], e["y_max"]) == (0.2, -0.1, -0.3, 0.4)  # inverted range kept as numpy's uniform takes it
    assert not e["ensure_valid"]
    e = _one(x_range=(-0.2, 0.1), y_range=(-0.3, 0.4))
    assert (e["x_min"], e["x_max"], e["y_min"], e["y_max"]) == (-0.2 + 0.03, 0.1 - 0.03, -0.3 + 0.03, 0.4 - 0.03) and e["ensure_valid"]
    assert (e["qpos_adr"], e["body"], e["radius"], e["bottom"], e["top"]) == (9, -1, 0.03, -0.02, 0.02)


def test_lowering_rotation_forms_and_axes():
    assert _one()["rot"] == [(0.0, 2 * math.pi)] and _one()["axis"] == 2
    assert _one(rotation=0.7)["rot"] == [(0.7, 0.7)]
    assert _one(rotation=(0.5, -0.25))["rot"] == [(-0.25, 0.5)]
    assert _one(rotation=[(0.1, 0.2), (1.0, 0.5), [3, 4]])["rot"] == [(0.1, 0.2), (0.5, 1.0), (3.0, 4.0)]
    assert [_one(rotation_axis=a)["axis"] for a in "xyz"] == [0, 1, 2]


def test_lowering_reference_offsets_and_composites():
    c = SequentialCompositeSampler("C")
    c.append_sampler(UniformRandomSampler("A", mujoco_objects="a", reference_pos=(0.1, 0.2, 0.8), z_offset=0.01))
    c.append_sampler(UniformRandomSampler("B", mujoco_objects="b", z_offset=0.005), sample_args={"reference": "a"})
    c.append_sampler(UniformRandomSampler("C2", mujoco_objects="c"), sample_args={"reference": "b", "on_top": False})
    names, (a, b, cc) = lower(c, OBJ)
    assert names == ["a", "b", "c"]
    assert (a["ref"], a["base"], a["ref_dz"], a["bottom_dz"], a["z_offset"]) == (-1, (0.1, 0.2, 0.8), 0.0, -0.02, 0.01)
    assert (b["ref"], b["base"], b["ref_dz"], b["bottom_dz"]) == (0, (0.0, 0.0, 0.0), 0.02, -0.025)  # on top of a: + a's top
    assert (cc["ref"], cc["ref_dz"], cc["bottom_dz"]) == (1, 0.0, 0.0)  # on_top False: neither offset
    c2 = SequentialCompositeSampler("V")
    c2.append_sampler(UniformRandomSampler("A", mujoco_objects=["a", "b"]), sample_args={"reference": (1, 2, 3), "on_top": False})
    c2.hide("c")
    names, (a, b, h) = lower(c2, OBJ)
    assert names == ["a", "b", "c"] and a["base"] == b["base"] == (1.0, 2.0, 3.0) and a["ref"] == -1 and a["bottom_dz"] == 0.0
    assert (h["x_min"], h["x_max"], h["rot"], h["z_offset"], h["ensure_valid"], h["bottom_dz"]) == (-10, -20, [(0.0, 0.0)], 10.0, False, -0.05)


def test_lowering_errors():
    with pytest.raises(ValueError, match="unknown object"):
        lower(UniformRandomSampler("S", mujoco_objects=["a", "zz"]), OBJ)
    with pytest.raises(ValueError, match="no sampler"):
        lower(UniformRandomSampler("S", mujoco_objects=["a", "b"]), OBJ)
    c = SequentialCompositeSampler("C")
    c.append_sampler(UniformRandomSampler("A", mujoco_objects="a"))
    c.append_sampler(UniformRandomSampler("B", mujoco_objects=["b", "c"]), sample_args={"reference": "c"})
    with pytest.raises(ValueError, match="not placed before"):
        lower(c, OBJ)
    inner = SequentialCompositeSampler("I")
    inner.append_sampler(UniformRandomSampler("A", mujoco_objects=["a", "b", "c"]))
    outer = SequentialCompositeSampler("O")
    outer.append_sampler(inner)
    outer.append_sampler(UniformRandomSampler("A2"))
    outer.samplers["A2"].add_objects("a")  # past append_sampler's check
    with pytest.raises(ValueError, match="already been sampled"):
        lower(outer, OBJ)


def test_sincos_is_within_an_ulp_of_numpy():
    rng = np.random.default_rng(0)
    xs = np.concatenate([rng.uniform(-20, 20, 4000), np.linspace(-4 * np.pi, 4 * np.pi, 2001), [0.0, np.pi / 4, -np.pi / 2]])
    for x in xs:
        s, c = sincos(x)
        assert abs(s - np.sin(x)) <= max(np.spacing(abs(np.sin(x))), 2.0 ** -60), x  # absolute near the zeros: two-part reduction
        assert abs(c - np.cos(x)) <= max(np.spacing(abs(np.cos(x))), 2.0 ** -60), x


def _table_samplers():
    """(sampler, objects) covering every option; the near-impossible one makes many tries"""
    out = []
    out.append(UniformRandomSampler("U", mujoco_objects=["a", "b", "c"], x_range=(-0.1, 0.1), y_range=(0.1, -0.1), rotation=None,
                                    reference_pos=(0.0, 0.0, 0.8), z_offset=0.01))
    out.append(UniformRandomSampler("X", mujoco_objects=["a", "b", "c"], x_range=(-0.08, 0.08), y_range=(-0.08, 0.08), rotation=(0.2, -0.4),
                                    rotation_axis="x", ensure_object_boundary_in_range=False))
    c = SequentialCompositeSampler("C")
    c.append_sampler(UniformRandomSampler("A", mujoco_objects="a", x_range=(-0.02, 0.02), y_range=(-0.02, 0.02), rotation=[(0, 0.5), (2, 3)],
                                          rotation_axis="y", reference_pos=(0.1, -0.1, 0.8), z_offset=0.01))
    c.append_sampler(UniformRandomSampler("B", mujoco_objects="b", rotation=1.25, ensure_object_boundary_in_range=False),
                     sample_args={"reference": "a"})
    c.hide("c")
    out.append(c)
    d = SequentialCompositeSampler("D")
    d.append_sampler(UniformRandomSampler("A", mujoco_objects=["a", "b"], x_range=(-0.045, 0.045), y_range=(-0.045, 0.045),
                                          ensure_object_boundary_in_range=False), sample_args={"reference": (0.0, 0.0, 0.8)})
    d.append_sampler(UniformRandomSampler("C", mujoco_objects="c", x_range=(0, 0.01), ensure_object_boundary_in_range=False),
                     sample_args={"reference": "b", "on_top": False})
    out.append(d)
    return out


@pytest.mark.parametrize("k", range(4))
def test_restatement_equals_the_reference_loop_given_the_same_uniforms(k):
    sampler = _table_samplers()[k]
    names, entries = lower(sampler, OBJ)
    for env in range(6):
        mine = place_env(entries, 1234567, 3, env)
        try:
            ref = reference_sample(sampler, OBJ, PhiloxStream(1234567, 3, env))
        except RandomizationError:
            assert any(t < 0 for *_, t in mine)
            continue
        assert all(t >= 0 for *_, t in mine)
        for name, (pos, quat, _) in zip(names, mine):
            rp, rq, _ = ref[name]
            assert [float(v) for v in pos] == [float(v) for v in rp], (name, pos, rp)  # positions: bit for bit
            np.testing.assert_allclose(quat, rq, rtol=0, atol=2.3e-16)  # sin / cos: the library's sequence vs libm, an ulp


def test_restatement_validity_and_failure():
    s = UniformRandomSampler("S", mujoco_objects=["a", "b"], x_range=(0, 0.001), y_range=(0, 0.001), ensure_object_boundary_in_range=False)
    _, entries = lower(s, {k: OBJ[k] for k in "ab"})
    res = place_values(entries, [0, 1], 9, 0)
    assert res["warn"].tolist() == [1024, 1024] and (res["tries"][:, 1] == -1).all() and (res["tries"][:, 0] == 0).all()
    s = UniformRandomSampler("S", mujoco_objects=["a", "b", "c"], x_range=(-0.12, 0.12), y_range=(-0.12, 0.12))
    _, entries = lower(s, OBJ)
    res = place_values(entries, range(20), 5, 1)
    assert (res["warn"] == 0).all() and res["tries"].max() > 0
    for e in range(20):
        for i in range(3):
            for j in range(i):
                d = np.hypot(*(res["pos"][e, i, :2] - res["pos"][e, j, :2]))
                assert d > OBJ["abc"[i]]["radius"] + OBJ["abc"[j]]["radius"]


# ---- the tasks, through the host layer on the CPU stand-in
def _make(task, sampler, n=3, **kw):
    return suite.make(task, robots="Panda", num_envs=n, seed=4, sim_cls=PlacementOracleSim, precision="f64",
                      placement_initializer=sampler, **kw)


def _cube_sampler(objs, half=0.1, **kw):
    return UniformRandomSampler("S", mujoco_objects=objs, x_range=(-half, half), y_range=(-half, half), reference_pos=(0, 0, 0.8),
                                z_offset=0.01, **kw)


@pytest.mark.parametrize("task, names", [("Lift", ["cube"]), ("Stack", ["cubeA", "cubeB"]), ("NutAssembly", ["SquareNut", "RoundNut"]),
                                         ("NutAssemblyRound", ["SquareNut", "RoundNut"]), ("NutAssemblySingle", ["SquareNut", "RoundNut"])])
def test_free_joint_tasks_place_through_the_host_layer(task, names):
    env = _make(task, _cube_sampler(None, half=0.1 if "cube" in names[0] else 0.4))
    assert env.placement_initializer.mujoco_objects == names and env._placement_names == names
    _, entries = lower(env.placement_initializer, env._placement_objects())
    q = env._reset_qpos.numpy()
    res = place_values(entries, range(3), env._place_seed, 0)
    parked = getattr(env, "single_object_mode", 0)
    for i, name in enumerate(names):
        a = entries[i]["qpos_adr"]
        rows = q[:, a:a + 7]
        want = np.concatenate([res["pos"][:, i], res["quat"][:, i]], axis=1)
        if parked == 2 and i != env.nut_id:
            assert (rows[:, :3] == 10.0).all()
        elif parked == 1:
            sel = env._sel_draw.numpy()
            assert all(np.array_equal(rows[e], want[e]) for e in range(3) if sel[e] == i)
        else:
            assert np.array_equal(rows, want)
    assert env.sim.place_calls[-1][1:] == (env._place_seed, 0)
    # a masked reset places the masked environments only, with the next counter
    before = env.sim.qpos.clone()
    m = torch.tensor([False, True, False])
    env.reset(mask=m)
    assert env.sim.place_calls[-1][2] == 1 and env.sim.place_calls[-1][0].tolist() == [0, 1, 0]
    assert torch.equal(env.sim.qpos[[0, 2]], before[[0, 2]])
    assert int(env.sim.warn.abs().max()) == 0


def test_door_places_its_pose_overrides():
    s = UniformRandomSampler("S", x_range=(0.05, 0.1), y_range=(-0.02, 0.02), rotation=(-1.8, -1.3), ensure_object_boundary_in_range=False,
                             reference_pos=(-0.2, -0.35, 0.8))
    env = _make("Door", s)
    _, entries = lower(s, env._placement_objects())
    (pm, qm), (pf, qf) = env._door_ov
    res = place_values(entries, range(3), env._place_seed, 0, ov_local={0: [env._frame_local]})
    for e in range(3):
        (p0, q0), (p1, q1) = res["ov"][0][e]
        assert pm[e].tolist() == [float(v) for v in p0] and qm[e].tolist() == [float(v) for v in q0]
        assert pf[e].tolist() == [float(v) for v in p1] and qf[e].tolist() == [float(v) for v in q1]
    assert pm[:, 2].tolist() == [0.8 + 0.3] * 3
    # the frame stays where the default path puts it relative to the door
    yaw = 2 * np.arctan2(qm[:, 3].numpy(), qm[:, 0].numpy())
    lp = env._frame_local[0]
    np.testing.assert_allclose(pf[:, 0].numpy(), pm[:, 0].numpy() + np.cos(yaw) * lp[0] - np.sin(yaw) * lp[1], atol=1e-15)


def test_impossible_sampler_sets_warn_bit_1024_after_the_reset():
    s = UniformRandomSampler("S", x_range=(0, 0.001), y_range=(0, 0.001), ensure_object_boundary_in_range=False, reference_pos=(0, 0, 0.8))
    env = _make("Stack", s, n=2)
    assert env.sim.warn.tolist() == [1024, 1024] and 1024 in SIM_WARN_BITS
    ok = _make("Stack", _cube_sampler(None), n=2)
    assert ok.sim.warn.tolist() == [0, 0]


def test_task_level_errors():
    with pytest.raises(ValueError, match="door_placement"):
        _make("Door", UniformRandomSampler("S"), door_placement=(0.08, 0.0, -1.7))
    with pytest.raises(NotImplementedError):
        _make("Lift", _cube_sampler(None), per_env_cube_size=True)
    with pytest.raises(NotImplementedError):
        _make("PickPlace", _cube_sampler(None))
    c = SequentialCompositeSampler("C")
    c.append_sampler(_cube_sampler("cubeA"))
    with pytest.raises(ValueError, match="no sampler"):
        _make("Stack", c)
    c = SequentialCompositeSampler("C")
    c.append_sampler(_cube_sampler(["cube", "mug"]))
    with pytest.raises(ValueError, match="unknown object"):
        _make("Lift", c)


def test_stack_composite_on_top_of_cube_b():
    c = SequentialCompositeSampler("C")
    c.append_sampler(_cube_sampler("cubeB"))
    c.append_sampler(UniformRandomSampler("OnB", mujoco_objects="cubeA", ensure_object_boundary_in_range=False,
                                          ensure_valid_placement=False), sample_args={"reference": "cubeB"})
    env = _make("Stack", c)
    q = env._reset_qpos.numpy()
    A, B = env.cubeA_qadr, env.cubeB_qadr
    assert np.array_equal(q[:, A:A + 2], q[:, B:B + 2])
    np.testing.assert_allclose(q[:, A + 2], q[:, B + 2] + env.half["B"][2] + env.half["A"][2], rtol=0, atol=1e-15)


def test_default_path_is_untouched():
    a = suite.make("Lift", robots="Panda", num_envs=2, seed=4, sim_cls=PlacementOracleSim, precision="f64")
    assert a.placement_initializer is None and a.sim.place_calls == []
