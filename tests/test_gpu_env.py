"""GPU: batched env API (make / reset / step / _get_observations) against the oracle's env step."""
import numpy as np
import pytest

import os

from tests.schedules import make_env
from tests.util import ROOT, load

pytestmark = pytest.mark.gpu


def _expected_obs(model, o, env):
    """observation row recomputed from oracle arrays with the reference's formulas (robots/robot.py:347-484,
    manipulation/lift.py:371-397)"""
    qp, qv = env._ref_joint_pos_indexes, env._ref_joint_vel_indexes
    jp = o.qpos[qp]
    site = env.eef_site_id
    M = o.site_xmat[site].reshape(3, 3)
    # mat2quat with w >= 0, xyzw
    tr = np.trace(M)
    w = np.sqrt(max(0.0, 1 + tr)) / 2
    x = (M[2, 1] - M[1, 2]) / (4 * w); y = (M[0, 2] - M[2, 0]) / (4 * w); z = (M[1, 0] - M[0, 1]) / (4 * w)
    bq = o.xquat[env.eef_body_id]
    cq = o.xquat[env.cube_body_id]
    return np.concatenate([
        jp, np.cos(jp), np.sin(jp), o.qvel[qv], o.qacc[qv], o.site_xpos[site], bq[[1, 2, 3, 0]], [x, y, z, w],
        o.qpos[env._ref_gripper_joint_pos_indexes], o.qvel[env._ref_gripper_joint_vel_indexes],
        o.xpos[env.cube_body_id], cq[[1, 2, 3, 0]], o.xpos[env.cube_body_id] - o.site_xpos[site]])


def test_env_api_and_obs_parity():
    import torch

    import robosuite_b200 as suite
    from oracle.pyoracle import CtrlCfg as OCfg
    from oracle.pyoracle import Oracle
    from robosuite_b200 import controller_config as cc
    from robosuite_b200.mjcf.compiler import pack_model

    n = 6
    env = suite.make("Lift", robots="Panda", num_envs=n, seed=3, has_renderer=False, has_offscreen_renderer=False,
                     use_camera_obs=False, horizon=5, reward_shaping=True)
    assert env.action_dim == 7 and env.obs_dim == 60
    low, high = env.action_spec
    assert np.all(low == -1) and np.all(high == 1)
    obs = env._get_observations()
    assert obs["robot0_proprio-state"].shape == (n, 50) and obs["object-state"].shape == (n, 10)
    assert list(obs.keys())[:3] == ["robot0_joint_pos", "robot0_joint_pos_cos", "robot0_joint_pos_sin"]
    model = env.model
    q0 = env.sim.qpos.cpu().numpy().astype(np.float64)
    # reset distribution sanity (lift.py:311-336): cube on the table within +-3 cm
    a = env.cube_qadr
    assert np.all(np.abs(q0[:, a:a + 2]) <= 0.03 + 1e-6) and np.allclose(q0[:, a + 2], 0.81 + env.cube_half_height, atol=1e-6)
    oracles = []
    for e in range(n):
        o = Oracle(pack_model(model))
        o.ctrl_setup(cc.resolve(model, cc.default_composite_config(), OCfg))
        o.qpos[:] = q0[e]
        o.forward()
        o.ctrl_reset()
        oracles.append(o)
    # reset observation = forced update at the reset state
    flat = env.flat_obs().cpu().numpy().astype(np.float64)
    for e in range(n):
        assert np.abs(flat[e] - _expected_obs(model, oracles[e], env)).max() < 2e-5
    rng = np.random.default_rng(0)
    for t in range(5):
        act = rng.uniform(-1, 1, size=(n, 7))
        obs, rew, done, info = env.step(torch.as_tensor(act))
        flat = env.flat_obs().cpu().numpy().astype(np.float64)
        for e in range(n):
            o = oracles[e]
            # observables sample on the last substep of the control step (poses of its step1, qpos/qvel after its step2)
            o.env_step(act[e], 25)
            exp = _expected_obs(model, o, env)
            err = np.abs(flat[e] - exp)
            err[28:35] /= max(1.0, np.abs(exp[28:35]).max())  # joint_acc: relative
            assert err.max() < 5e-4, (t, e, err.argmax(), err.max())
            # shaped reward from the last step1 poses
            dist = np.linalg.norm(o.xpos[env.cube_body_id] - o.site_xpos[env.eef_site_id])
            lifted = o.xpos[env.cube_body_id][2] > 0.84
            expect = 2.25 if lifted else (1 - np.tanh(10 * dist))
            assert abs(float(rew[e]) - expect / 2.25) < 1e-3
    assert bool(done.all())
    with pytest.raises(ValueError):
        env.step(torch.zeros((n, 7)))
    env.reset()
    assert not bool(env.done.any())
    env.close()


def test_stack_sawyer_joint_velocity_env_parity():
    """BASELINE config 3 path: Stack / Sawyer / JOINT_VELOCITY + GRIP through the env API vs the oracle"""
    import torch

    import robosuite_b200 as suite
    from oracle.pyoracle import CtrlCfg as OCfg
    from oracle.pyoracle import Oracle
    from robosuite_b200 import controller_config as cc
    from robosuite_b200.mjcf.compiler import pack_model

    n = 6
    cfg = cc.refactor_composite_controller_config(cc.load_part_controller_config("JOINT_VELOCITY"), "Sawyer", ["right"])
    # The Sawyer model has two knife-edge coincidences that make constraint activation depend on the last bit of rounding
    # (in ANY engine): the l0 collision sphere exactly touches the rim of the base cylinder (dist = -5.6e-17 in fp64), and
    # the gripper's initial qpos equals its joint limit.  De-degenerate both in the model used by BOTH sides.
    model = load("Stack_Sawyer")
    model.geom_size[model.names["geom"].index("robot0_link0_collision"), 0] -= 1e-5
    model.jnt_range[[model.names["joint"].index("gripper0_right_l_finger_joint"),
                     model.names["joint"].index("gripper0_right_r_finger_joint")]] += np.array([-1e-6, 1e-6])
    env = suite.make("Stack", robots="Sawyer", num_envs=n, seed=5, controller_configs=cfg, horizon=100, reward_shaping=True,
                     model=model)
    assert env.action_dim == 8 and env.obs_dim == 73
    obs = env._get_observations()
    assert obs["object-state"].shape == (n, 23) and obs["robot0_proprio-state"].shape == (n, 50)
    model = env.model
    q0 = env.sim.qpos.cpu().numpy().astype(np.float64)
    # placement: cubes on the table, not overlapping (stack.py:357-388)
    a, b = env.cubeA_qadr, env.cubeB_qadr
    assert np.all(np.linalg.norm(q0[:, a:a + 2] - q0[:, b:b + 2], axis=1) > np.linalg.norm(env.half["A"][:2]) + np.linalg.norm(env.half["B"][:2]))
    oracles = []
    for e in range(n):
        o = Oracle(pack_model(model))
        o.ctrl_setup(cc.resolve(model, cfg, OCfg, gripper="rethink"))
        o.qpos[:] = q0[e]; o.forward(); o.ctrl_reset()
        oracles.append(o)
    rng = np.random.default_rng(0)
    for t in range(4):
        act = rng.uniform(-1, 1, size=(n, 8))
        obs, rew, done, info = env.step(torch.as_tensor(act))
        for e in range(n):
            oracles[e].env_step(act[e], 25)
    qd = env.sim.qpos.cpu().numpy().astype(np.float64)
    eq = max(np.abs(qd[e] - oracles[e].qpos).max() / np.abs(oracles[e].qpos).max() for e in range(n))
    print("Stack/Sawyer/JOINT_VELOCITY 100 substeps: qpos rel err %.3g" % eq)
    assert eq < 1e-4
    assert int(env.sim.warn.abs().max()) == 0
    # staged reward pieces from the oracle's last step1 poses
    for e in range(n):
        o = oracles[e]
        dist = np.linalg.norm(o.site_xpos[env.eef_site_id] - o.xpos[env.cubeA_body_id])
        # (poses of the oracle are one substep ahead only after a forward; env_step leaves step1 poses of the last substep)
        r_reach = (1 - np.tanh(10 * dist)) * 0.25
        assert abs(float(rew[e]) * 2.0 - r_reach) < 5e-3 or float(rew[e]) * 2.0 >= r_reach - 5e-3
    env.close()


def _quat_xyzw_wpos_from_mat(M):
    """T.mat2quat semantics (transform_utils.py:317-355): unit quaternion of M with w >= 0, (x, y, z, w)"""
    from scipy.spatial.transform import Rotation

    q = Rotation.from_matrix(M).as_quat()  # x, y, z, w
    return -q if q[3] < 0 else q


def _quat2mat_wxyz(q):
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def _object_obs(env, o, cache, task):
    """object-state row from oracle arrays with the reference's sensor ORDER semantics: `{obj}_to_eef_pos/quat` are
    evaluated before `{obj}_pos/quat` and read the cached values of the previous sample (zeros on an empty cache)"""
    eef_pos = o.site_xpos[env.eef_site_id].copy()
    Re = _quat2mat_wxyz(o.xquat[env.eef_body_id])
    out = []
    if task == "Door":
        d, h = o.xpos[env.door_body_id], o.site_xpos[env.door_handle_site_id]
        out = [d, h, [o.qpos[env.hinge_qpos_addr]], d - eef_pos, h - eef_pos, [o.qpos[env.handle_qpos_addr]]]
        return np.concatenate(out)
    names = [env.nut_names[i] for i in env.active] if task.startswith("Nut") else list(env.obj_names)
    for nme in names:
        b = env.obj_body_id[nme]
        if nme in cache:
            p_prev, q_prev = cache[nme]  # q xyzw
            rel_pos = Re.T @ (p_prev - eef_pos)
            Ro = _quat2mat_wxyz(q_prev[[3, 0, 1, 2]])
            rel_q = _quat_xyzw_wpos_from_mat(Re.T @ Ro)
        else:
            rel_pos, rel_q = np.zeros(3), np.zeros(4)
        p, q = o.xpos[b].copy(), o.xquat[b][[1, 2, 3, 0]].copy()
        cache[nme] = (p, q)
        out += [rel_pos, rel_q, p, q]
    return np.concatenate(out)


@pytest.mark.parametrize("task,obs_dim", [("Door", 64), ("NutAssemblyRound", 64), ("PickPlace", 106)])
def test_other_task_envs_obs_and_reward(task, obs_dim):
    """Door / NutAssemblyRound / PickPlace through the env API: observation layout incl. the one-sample lag of the
    object-in-gripper poses, state parity after 3 control steps, sparse/shaped reward pieces from the oracle poses"""
    import torch

    import robosuite_b200 as suite
    from oracle.pyoracle import CtrlCfg as OCfg
    from oracle.pyoracle import Oracle
    from robosuite_b200 import controller_config as cc
    from robosuite_b200.mjcf.compiler import pack_model

    n = 3
    env = suite.make(task, robots="Panda", num_envs=n, seed=11, horizon=50, reward_shaping=True)
    assert env.action_dim == 7 and env.obs_dim == obs_dim, (env.action_dim, env.obs_dim)
    model = env.model
    q0 = env.sim.qpos.cpu().numpy().astype(np.float64)
    oracles, caches = [], []
    for e in range(n):
        o = Oracle(pack_model(model))
        o.ctrl_setup(cc.resolve(model, cc.default_composite_config(), OCfg))
        if task == "Door":  # the door pose is drawn per environment and reset (door.py:417-427): the oracle gets it as model constants
            assert env.door_pose is not None
            P, Q = (t.cpu().numpy().astype(np.float64) for t in env.door_pose)
            o.set_body_pose(model.names["body"].index("Door_main"), P[e], Q[e])
        o.qpos[:] = q0[e]; o.forward(); o.ctrl_reset()
        oracles.append(o); caches.append({})
    if task == "Door":
        assert np.abs(P[0] - P[1]).max() > 1e-4  # really per environment
    flat = env.flat_obs().cpu().numpy().astype(np.float64)
    for e in range(n):
        exp = _object_obs(env, oracles[e], caches[e], task)
        assert np.abs(flat[e, 50:] - exp).max() < 2e-5, (task, "reset", np.abs(flat[e, 50:] - exp).argmax())
    rng = np.random.default_rng(1)
    for t in range(3):
        act = rng.uniform(-1, 1, size=(n, 7))
        obs, rew, done, info = env.step(torch.as_tensor(act))
        flat = env.flat_obs().cpu().numpy().astype(np.float64)
        for e in range(n):
            o = oracles[e]
            o.env_step(act[e], 25)
            exp = _object_obs(env, o, caches[e], task)
            err = np.abs(flat[e, 50:] - exp)
            # (PickPlace: mesh objects settling on the bin floor amplify fp32 rounding in their orientation)
            assert err.max() < (3e-3 if task == "PickPlace" else 1e-3), (task, t, e, int(err.argmax()), float(err.max()))
            # reaching term of the shaped reward from the oracle's poses after the step
            eef = o.site_xpos[env.eef_site_id]
            if task == "Door":
                expect = 0.25 * (1 - np.tanh(10 * np.linalg.norm(o.site_xpos[env.door_handle_site_id] - eef))) \
                    + np.clip(0.25 * abs(o.qpos[env.handle_qpos_addr] / (0.5 * np.pi)), -0.25, 0.25)
                assert abs(float(rew[e]) - expect) < 2e-3, (float(rew[e]), expect)
            elif task.startswith("Nut"):
                d = min(np.linalg.norm(o.site_xpos[s] - eef) for s in env.object_site_ids)
                assert float(rew[e]) >= (1 - np.tanh(10 * d)) * 0.1 - 2e-3
            else:
                d = min(np.linalg.norm(o.xpos[env.obj_body_id[nm]] - eef) for nm in env.obj_names)
                assert float(rew[e]) * 4.0 >= (1 - np.tanh(10 * d)) * 0.1 - 2e-3
    qd = env.sim.qpos.cpu().numpy().astype(np.float64)
    eq = max(np.abs(qd[e] - oracles[e].qpos).max() / np.abs(oracles[e].qpos).max() for e in range(n))
    print(task, "75 substeps through the env API: qpos rel err %.3g, warn %s" % (eq, env.sim.warn.tolist()))
    assert eq < 2e-3
    assert int(env.sim.warn.abs().max()) == 0
    env.close()


def test_batched_gym_wrapper_autoreset():
    """GymWrapper semantics (wrappers/gym_wrapper.py:26-180) on the batch: key order, 5-tuple, reset inside step"""
    import torch

    import robosuite_b200 as suite
    from robosuite_b200.wrappers import BatchedGymWrapper

    n = 4
    env = BatchedGymWrapper(suite.make("Lift", robots="Panda", num_envs=n, seed=2, horizon=3))
    obs, info = env.reset(seed=7)
    assert obs.shape == (n, 60) and info == {}
    d = env.env._get_observations()
    assert torch.equal(obs[:, :10], d["object-state"]) and torch.equal(obs[:, 10:], d["robot0_proprio-state"])
    for t in range(3):
        obs, rew, term, trunc, info = env.step(torch.zeros((n, 7), device=obs.device))
        assert rew.shape == (n,) and term.shape == (n,) and not bool(trunc.any())
    assert bool(term.all()) and "final_observation" in info
    assert int(env.env.timestep.max()) == 0 and not bool(env.env.done.any())  # every environment started a new episode
    # the observation handed back is the reset observation: cube back on the table
    assert torch.allclose(obs[:, 2], torch.full((n,), 0.83, device=obs.device), atol=5e-3)
    obs, rew, term, trunc, info = env.step(torch.zeros((n, 7), device=obs.device))  # stepping continues without an explicit reset
    assert not bool(term.any())
    env.close()


@pytest.mark.gpu
def test_device_joint_velocity_replays_reference_class_golden():
    """Device (fp64) replay of tests/golden/jv_golden.npz - actions, torques and trajectories recorded from the reference's own
    JointVelocityController methods (tools/gen_jv_golden.py) on Stack / Sawyer: the arm-torque part of `ctrl` per control step and the
    state after every control step.  Tolerance: 1e-6 absolute on qpos over 150 substeps of contact-free motion with a saturating PID
    (the controller is a discontinuous map at the clip, so agreement here means the same branch was taken on every substep)."""
    import torch

    import robosuite_b200 as suite
    from robosuite_b200 import controller_config as cc
    from tests.util import dedegenerate_sawyer

    g = np.load(os.path.join(ROOT, "tests", "golden", "jv_golden.npz"))
    n, n_steps = g["actions"].shape[:2]
    nsub = int(g["nsub"])
    cfg = cc.refactor_composite_controller_config(cc.load_part_controller_config("JOINT_VELOCITY"), "Sawyer", ["right"])
    env = suite.make("Stack", robots="Sawyer", num_envs=n, seed=1, controller_configs=cfg, horizon=1000,
                     model=dedegenerate_sawyer(load("Stack_Sawyer")), precision="f64")
    env.reset_to(torch.as_tensor(g["qpos0"]))
    worst_q, worst_v, worst_u = 0.0, 0.0, 0.0
    for t in range(n_steps):
        env.step(torch.as_tensor(g["actions"][:, t]))
        q, v = env.sim.qpos.cpu().numpy(), env.sim.qvel.cpu().numpy()
        u = env.sim.ctrl.cpu().numpy()
        worst_q = max(worst_q, np.abs(q - g["qpos"][:, t]).max())
        worst_v = max(worst_v, np.abs(v - g["qvel"][:, t]).max())
        worst_u = max(worst_u, np.abs(u - g["ctrl"][:, (t + 1) * nsub - 1]).max())
    print("JV golden replay on the device: |dq| %.3g |dv| %.3g |dctrl| %.3g" % (worst_q, worst_v, worst_u))
    assert worst_q < 1e-6 and worst_v < 1e-4 and worst_u < 1e-3
    assert int(env.sim.warn.abs().max()) == 0
    env.close()


@pytest.mark.parametrize("task,robot,ctrl", [("Stack", "Sawyer", "JOINT_VELOCITY"), ("Door", "Panda", "OSC_POSE"),
                                             ("PickPlace", "Panda", "OSC_POSE"), ("NutAssemblyRound", "Panda", "OSC_POSE")])
def test_unit_queue_mode_matches_pipeline_on_task_envs(task, robot, ctrl):
    """mode 2 (persistent unit-queue kernel) against mode 1 (phase pipeline) through the env API on the other BASELINE tasks: tiered
    layouts (Door, PickPlace), the JOINT_VELOCITY controller, a 33-dof model.  Same device functions, same per-environment data ->
    bit-identical states and observations (OSC evaluated inside the tail in both, B2S_CTRL_SPLIT=0: the thread-per-environment
    controller kernel of the pipeline orders its fp64 sums differently)"""
    import torch

    from robosuite_b200 import controller_config as cc

    n, steps = 24, 5
    kw = {}
    if ctrl != "OSC_POSE":
        kw["controller_configs"] = cc.refactor_composite_controller_config(cc.load_part_controller_config(ctrl), robot, ["right"])
    out = []
    for mode in (1, 2):
        env = make_env(task, n, mode, 5, ctrl_split=False, robots=robot, horizon=10 ** 6, **kw)
        gen = torch.Generator(device=env.device)
        gen.manual_seed(9)
        for t in range(steps):
            act = torch.rand((n, env.action_dim), generator=gen, device=env.device, dtype=env.dtype) * 2 - 1
            act[: n // 2, 2] = -1.0  # half of the arms push down: contacts, EPA, large-tier environments
            env.step(act)
        torch.cuda.synchronize()
        assert int(env.sim.warn.abs().max()) == 0
        out.append((env.sim.qpos.clone(), env.sim.qvel.clone(), env.flat_obs().clone()))
        env.close()
    for a, b in zip(out[0], out[1]):
        assert torch.isfinite(b).all() and torch.equal(a, b)
