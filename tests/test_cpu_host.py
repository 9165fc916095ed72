"""CPU-only tests: MJCF compiler, model blob, oracle known-answer tests, C-ABI symbols, multi-process plumbing."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from tests.util import ROOT, lift_states, load


def _oracle(model):
    from oracle.pyoracle import Oracle
    from robosuite_b200.mjcf.compiler import pack_model

    return Oracle(pack_model(model))


# ------------------------------------------------------------------------------------------------ compiler
def test_compiled_model_sizes_match_reference_survey():
    """sizes the reference's own composer + engine report for these models (SURVEY.md section 8a table)"""
    exp = {"Lift_Panda": (26, 10, 16, 15, 9, 90, 9), "Stack_Sawyer": (37, 11, 23, 21, 9, 105, 10),
           "NutAssemblyRound_Panda": (29, 11, 23, 21, 9, 120, 14), "Door_Panda": (29, 11, 11, 11, 9, 102, 10),
           "PickPlace_Panda": (34, 13, 37, 33, 9, 126, 15)}
    for name, (nbody, njnt, nq, nv, nu, ngeom, nsite) in exp.items():
        m = load(name)
        assert (m.nbody, m.njnt, m.nq, m.nv, m.nu, m.ngeom, m.nsite) == (nbody, njnt, nq, nv, nu, ngeom, nsite), name


def test_body_order_and_names():
    m = load("Lift_Panda")
    b = m.names["body"]
    assert b[:5] == ["world", "table", "left_eef_target", "right_eef_target", "robot0_base"]
    assert b[-1] == "cube_main" and m.names["actuator"][0] == "robot0_torq_j1"
    assert m.names["sensor"] == ["gripper0_right_force_ee", "gripper0_right_torque_ee"]


def test_box_inertia_from_geom():
    m = load("Lift_Panda")
    g = m.names["geom"].index("cube_g0")
    sx, sy, sz = m.geom_size[g]
    mass = 1000 * 8 * sx * sy * sz
    b = m.names["body"].index("cube_main")
    assert abs(m.body_mass[b] - mass) < 1e-12
    I = sorted(mass / 3 * np.array([sy * sy + sz * sz, sx * sx + sz * sz, sx * sx + sy * sy]), reverse=True)
    assert np.allclose(m.body_inertia[b], I)


def test_blob_roundtrip_and_fixture_stability():
    from robosuite_b200.mjcf.compiler import load_model, pack_model, save_model

    m = load("Lift_Panda")
    blob = pack_model(m)
    assert blob[:8] == b"B2SMODEL"
    import io
    buf = io.BytesIO()
    save_model(m, buf)
    buf.seek(0)
    assert pack_model(load_model(buf)) == blob


def test_compile_from_xml_needs_no_meshes_for_primitive_models():
    from robosuite_b200.mjcf.compiler import compile_mjcf

    xml = """<mujoco><option timestep="0.002" cone="elliptic" impratio="20"/><worldbody>
    <geom type="plane" size="1 1 .1"/>
    <body name="p" pos="0 0 1"><joint type="hinge" axis="0 1 0" name="h"/><geom type="sphere" size=".05" pos="0 0 -0.5" mass="1"/></body>
    <body name="c" pos="0.5 0 0.1"><freejoint name="f"/><geom type="box" size=".1 .1 .1" name="b"/></body>
    </worldbody><actuator><motor joint="h" name="m" ctrlrange="-1 1"/></actuator></mujoco>"""
    m = compile_mjcf(xml)
    assert (m.nq, m.nv, m.nu, m.npair) == (8, 7, 1, 3)


# ------------------------------------------------------------------------------------------------ oracle KATs
def _simple(xml):
    from robosuite_b200.mjcf.compiler import compile_mjcf

    m = compile_mjcf(xml)
    return m, _oracle(m)


def test_kat_pendulum_period():
    """small-angle period of a point-mass pendulum: T = 2 pi sqrt(l / g)"""
    xml = """<mujoco><option timestep="0.0005" cone="elliptic"/><worldbody><body pos="0 0 2">
    <joint type="hinge" axis="0 1 0"/><geom type="sphere" size=".001" pos="0 0 -1" mass="1" contype="0" conaffinity="0"/></body></worldbody></mujoco>"""
    m, o = _simple(xml)
    o.qpos[0] = 0.01
    zero = []
    prev = o.qpos[0]
    for i in range(6000):
        o.step()
        if prev > 0 >= o.qpos[0] or prev < 0 <= o.qpos[0]:
            zero.append(o.time)
        prev = o.qpos[0]
    period = 2 * np.mean(np.diff(zero))
    assert abs(period - 2 * np.pi * np.sqrt(1 / 9.81)) < 2e-3


def test_kat_free_fall_and_quaternion_integration():
    xml = """<mujoco><option timestep="0.001" cone="elliptic"/><worldbody><body pos="0 0 10"><freejoint/>
    <geom type="sphere" size=".1" mass="1" contype="0" conaffinity="0"/></body></worldbody></mujoco>"""
    m, o = _simple(xml)
    o.qvel[3:6] = [0, 0, 2.0]  # spin about z
    for _ in range(1000):
        o.step()
    t = 1.0
    assert abs(o.qpos[2] - (10 - 0.5 * 9.81 * t * t)) < 0.01  # semi-implicit Euler: O(h) error
    ang = 2 * np.arctan2(o.qpos[6], o.qpos[3])
    assert abs(ang - 2.0) < 1e-9 and abs(np.linalg.norm(o.qpos[3:7]) - 1) < 1e-12


def test_kat_box_rest_force_equals_weight():
    xml = """<mujoco><option timestep="0.002" cone="elliptic" impratio="20"/><worldbody><geom type="plane" size="2 2 .1"/>
    <body pos="0 0 0.1"><freejoint/><geom type="box" size=".1 .1 .1" mass="2"/></body></worldbody></mujoco>"""
    m, o = _simple(xml)
    for _ in range(1500):
        o.step()
    o.forward()
    cs = [c for c in o.contacts() if c["efc_address"] >= 0]
    assert len(cs) == 4
    f = o.efc("force")
    total = sum(f[c["efc_address"]] for c in cs)
    assert abs(total - 2 * 9.81) < 1e-3 * 2 * 9.81
    assert np.abs(o.qvel).max() < 1e-6
    # resting penetration is set by solref/solimp: small and negative
    assert all(-2e-3 < c["dist"] < 0 for c in cs)


def test_kat_friction_cone_threshold():
    """box on a tilted plane (via tilted gravity): sticks below mu, slides above (mu = 1)"""
    from robosuite_b200.mjcf.compiler import compile_mjcf

    for tilt, slides in ((0.6, False), (1.3, True)):
        xml = f"""<mujoco><option timestep="0.002" cone="elliptic" impratio="20" gravity="{9.81 * np.sin(np.arctan(tilt))} 0 {-9.81 * np.cos(np.arctan(tilt))}"/>
        <worldbody><geom type="plane" size="5 5 .1"/><body pos="0 0 0.1"><freejoint/><geom type="box" size=".1 .1 .1" mass="1"/></body></worldbody></mujoco>"""
        m = compile_mjcf(xml)
        o = _oracle(m)
        for _ in range(500):
            o.step()
        assert (abs(o.qvel[0]) > 0.5) == slides, (tilt, o.qvel[0])


def test_kat_position_actuator_forcerange_and_joint_limit():
    xml = """<mujoco><option timestep="0.002" cone="elliptic"/><worldbody><body><joint type="slide" axis="1 0 0" name="s" range="-0.1 0.1" damping="1"/>
    <geom type="sphere" size=".05" mass="1" contype="0" conaffinity="0"/></body></worldbody>
    <actuator><position joint="s" kp="1000" forcerange="-20 20" ctrlrange="-1 1" name="a"/></actuator></mujoco>"""
    m, o = _simple(xml)
    o.ctrl[0] = 1.0
    o.forward()
    assert abs(o.actuator_force[0] - 20.0) < 1e-12  # kp * (1 - 0) clamped to the force range
    for _ in range(2000):
        o.step()
    assert 0.1 < o.qpos[0] < 0.105  # held at the (soft) joint limit


def test_oracle_determinism_and_playback():
    """the reference's own property tests: same seed -> same state; open-loop playback is bit-identical
    (tests/test_environments/test_env_determinism.py:27-111, test_action_playback.py:17-70)"""
    from oracle.pyoracle import CtrlCfg
    from robosuite_b200 import controller_config as cc

    model = load("Lift_Panda")
    q, _ = lift_states(model, 1, seed=5)
    rng = np.random.default_rng(0)
    acts = 0.1 * rng.uniform(-1, 1, size=(20, 7))
    outs = []
    for rep in range(2):
        o = _oracle(model)
        o.ctrl_setup(cc.resolve(model, cc.default_composite_config(), CtrlCfg))
        o.qpos[:] = q[0]; o.forward(); o.ctrl_reset()
        for a in acts:
            o.env_step(a, 25)
        outs.append(np.concatenate([[o.time], o.qpos, o.qvel]))
    assert np.array_equal(outs[0], outs[1])


def test_gripper_lift_behaviour():
    """gripper tester of the reference (models/grippers/gripper_tester.py:111-235): close on the cube, lift, the cube must
    follow (height gain >= 0.01) - a contact / friction-cone behaviour check, here through OSC actions"""
    from oracle.pyoracle import CtrlCfg
    from robosuite_b200 import controller_config as cc

    model = load("Lift_Panda")
    o = _oracle(model)
    o.ctrl_setup(cc.resolve(model, cc.default_composite_config(), CtrlCfg))
    q, _ = lift_states(model, 1, seed=0)
    q[0, :7] = [0, np.pi / 16.0, 0.00, -np.pi / 2.0 - np.pi / 3.0, 0.00, np.pi - 0.2, np.pi / 4]
    q[0, 9:11] = 0
    q[0, 12:16] = [1, 0, 0, 0]
    o.qpos[:] = q[0]; o.forward(); o.ctrl_reset()
    cube = model.names["body"].index("cube_main")
    site = model.names["site"].index("gripper0_right_grip_site")
    z0 = None
    for t in range(120):
        o.step1()
        d = o.xpos[cube] - o.site_xpos[site]
        if z0 is None:
            z0 = o.xpos[cube][2]
        if t < 50:   # descend over the cube, gripper open
            a = np.concatenate([np.clip(d * 10, -1, 1), [0, 0, 0], [-1]])
        elif t < 70:  # close
            a = np.array([0, 0, 0, 0, 0, 0, 1.0])
        else:         # lift
            a = np.array([0, 0, 0.5, 0, 0, 0, 1.0])
        o.ctrl_run(a)
        o.step2()
        for _ in range(24):
            o.step1(); o.ctrl_run(None); o.step2()
    assert o.xpos[cube][2] - z0 > 0.01, o.xpos[cube][2] - z0


# ------------------------------------------------------------------------------------------------ C ABI
def test_c_abi_exports_every_declared_symbol():
    so = os.path.join(ROOT, "robosuite_b200", "libb2s.so")
    if not os.path.exists(so):
        from robosuite_b200 import build

        build.build()
    hdr = open(os.path.join(ROOT, "include", "b2s.h")).read()
    names = sorted(set(re.findall(r"\b(b2s_[a-z0-9_]+)\s*\(", hdr)))
    assert len(names) >= 18
    lib = ctypes.CDLL(so)  # loads without a GPU; no compute calls here
    for n in names:
        assert hasattr(lib, n), n


def test_create_without_gpu_fails_loudly():
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from robosuite_b200.engine import B2SError, BatchedSim

    with pytest.raises(B2SError):
        BatchedSim(load("Lift_Panda"), 2)


def test_controller_config_surface():
    from oracle.pyoracle import CtrlCfg
    from robosuite_b200 import controller_config as cc

    model = load("Lift_Panda")
    cfg = cc.load_composite_controller_config(None, "Panda")
    assert cfg["type"] == "BASIC" and cfg["body_parts"]["arms"]["right"]["type"] == "OSC_POSE"
    c = cc.resolve(model, cfg, CtrlCfg)
    assert c.n_arm == 7 and list(c.arm_dof)[:7] == list(range(7)) and c.n_grip == 2 and c.action_dim == 7
    assert model.names["site"][c.eef_site] == "gripper0_right_grip_site"
    bad = {"type": "BASIC", "body_parts": {"arms": {"right": {"type": "IK_POSE"}}}}
    with pytest.raises(NotImplementedError):
        cc.resolve(model, bad, CtrlCfg)


def test_switches_set_the_library_variables_and_restore_them():
    """tests/schedules.py's switches(): the requested values inside; on exit, also through an exception, an absent variable is absent
    again and a pre-existing value (here a user's B2S_GROUPS=4, itself set by an outer switches()) is back"""
    from tests.schedules import switches

    def now():
        return [os.environ.get(k) for k in ("B2S_NO_GJK_CACHE", "B2S_CTRL_SPLIT", "B2S_GROUPS")]

    outside = now()
    with switches(groups=4):
        assert now() == [None, None, "4"]
        with switches(gjk_cache=False, ctrl_split=False, groups=1):
            assert now() == ["1", "0", "1"]
        assert now() == [None, None, "4"]
        with pytest.raises(RuntimeError):
            with switches(gjk_cache=False, ctrl_split=False):
                assert now() == ["1", "0", None]
                raise RuntimeError("inside")
        assert now() == [None, None, "4"]
    assert now() == outside


# ------------------------------------------------------------------------------------------------ multi-process
_WORKER = r"""
import os, sys, torch, numpy as np
sys.path.insert(0, os.environ["B2S_ROOT"])
import torch.distributed as dist
from robosuite_b200.parallel import broadcast_model, allgather_obs, shard_range
from robosuite_b200.mjcf.compiler import pack_model
from tests.util import load
dist.init_process_group("gloo")
rank, world = dist.get_rank(), dist.get_world_size()
model = load("Lift_Panda") if rank == 0 else None
model = broadcast_model(model, src=0)
ref = load("Lift_Panda")
assert pack_model(model) == pack_model(ref)
lo, hi = shard_range(10, rank, world)
obs = torch.arange(lo * 3, hi * 3, dtype=torch.float32).reshape(hi - lo, 3)
g = allgather_obs(obs) if (hi - lo) * world == 10 else None
if g is not None:
    assert torch.equal(g, torch.arange(30, dtype=torch.float32).reshape(10, 3))
dist.barrier()
open(os.path.join(os.environ["B2S_OUT"], f"ok{rank}"), "w").write("ok")
"""


def test_two_process_model_broadcast_and_obs_allgather(tmp_path):
    script = tmp_path / "w.py"
    script.write_text(_WORKER)
    env = dict(os.environ, B2S_ROOT=ROOT, B2S_OUT=str(tmp_path))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                        "--master-port", "29543", str(script)], env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert (tmp_path / "ok0").exists() and (tmp_path / "ok1").exists()


def test_shard_range_partitions():
    from robosuite_b200.parallel import shard_range

    for n, w in ((65536, 8), (10, 3), (7, 8)):
        spans = [shard_range(n, r, w) for r in range(w)]
        assert spans[0][0] == 0 and spans[-1][1] == n and all(spans[i][1] == spans[i + 1][0] for i in range(w - 1))


def test_state_io_formats_roundtrip(tmp_path):
    """MjSimState.flatten layout and DataCollectionWrapper episode folders (binding_utils.py:221-249,
    wrappers/data_collection_wrapper.py:100-147)"""
    from robosuite_b200 import state_io as sio

    rng = np.random.default_rng(0)
    T, N, nq, nv, A = 5, 3, 16, 15, 7
    qpos, qvel, time = rng.normal(size=(T + 1, N, nq)), rng.normal(size=(T + 1, N, nv)), np.arange(T + 1) * 0.05
    states = np.stack([sio.flatten_state(time[t], qpos[t], qvel[t]) for t in range(T + 1)])
    assert states.shape == (T + 1, N, 1 + nq + nv) and np.all(states[2, :, 0] == 0.1)
    t2, q2, v2 = sio.unflatten_state(states[3], nq, nv)
    assert np.array_equal(q2, qpos[3]) and np.array_equal(v2, qvel[3]) and np.allclose(t2, 0.15)
    with pytest.raises(ValueError):
        sio.unflatten_state(states[0][:, :-1], nq, nv)
    actions = rng.uniform(-1, 1, size=(T, N, A))
    eps = sio.save_episodes(str(tmp_path), "Lift", "<mujoco/>", states, actions, successful=[True, False, False])
    assert len(eps) == N and sorted(os.listdir(eps[0])) == ["ep_meta.json", "model.xml", "state_0_0.npz"]
    raw = np.load(os.path.join(eps[1], "state_0_0.npz"), allow_pickle=True)  # the keys the reference writes
    assert set(raw.files) == {"states", "action_infos", "successful", "env"} and raw["states"].shape == (T + 1, 1 + nq + nv)
    ep = sio.load_episode(eps[0])
    assert ep["env"] == "Lift" and ep["successful"] and ep["model_xml"] == "<mujoco/>"
    assert np.array_equal(ep["states"], states[:, 0]) and np.array_equal(ep["actions"], actions[:, 0])


def test_error_classes_follow_the_reference_names():
    """utils/errors.py names; malformed MJCF -> XMLError; library failures -> SimulationError subclasses"""
    from robosuite_b200.engine import B2SError
    from robosuite_b200.errors import RandomizationError, SimulationError, XMLError, robosuiteError
    from robosuite_b200.mjcf.compiler import compile_mjcf

    assert issubclass(XMLError, robosuiteError) and issubclass(RandomizationError, robosuiteError)
    assert issubclass(B2SError, SimulationError) and issubclass(B2SError, RuntimeError)
    with pytest.raises(XMLError):
        compile_mjcf("<mujoco><worldbody>")
    with pytest.raises(XMLError):
        compile_mjcf("<robot/>")


def test_oracle_resets_diverged_state_like_mj_check():
    """mj_checkPos / mj_checkVel / mj_checkAcc: a non-finite or huge coordinate resets the data to the model defaults (time 0, warn bit
    32) instead of integrating garbage; the device engine mirrors this (tests/test_gpu_engine.py)"""
    model = load("Lift_Panda")
    q, _ = lift_states(model, 1, seed=5)
    o = _oracle(model)
    o.qpos[:] = q[0]
    for _ in range(3):
        o.step()
    assert o.time > 0 and o.geti("warn_flags") == 0
    o.qvel[2] = np.nan
    o.step()
    assert o.geti("warn_flags") & 32
    assert np.isfinite(o.qpos).all() and np.isfinite(o.qvel).all()
    assert abs(o.time - model.opt_timestep) < 1e-12  # the clock restarted, then one step was integrated from qpos0
    o2 = _oracle(model)
    o2.step()
    assert np.array_equal(o.qpos, o2.qpos)
    o.qvel[0] = 1e12  # huge, finite
    o.step()
    assert np.abs(o.qvel).max() < 1e3
