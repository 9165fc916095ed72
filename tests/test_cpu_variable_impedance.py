"""CPU: variable impedance (impedance_mode "variable" / "variable_kp") of OSC_POSE, OSC_POSITION and JOINT_POSITION.

  * controller_config.resolve: action_dim and BatchedMujocoEnv.action_spec for every kind and mode (OSC_POSITION's fixed mode
    has 4 bounds), scalar and vector limits broadcast to d (6 for OSC, n_arm for JOINT_POSITION), and the errors;
  * the gain restatement (tests/impedance_ref.py) against hand-computed gains: kp beyond its limits, a damping ratio beyond its
    limits, kp = 0 giving kd = 0;
  * the restatement against the oracle's controller, substep by substep, for both modes of kinds 1, 5 and 3 on the Panda and the
    Sawyer, on test_cpu_controllers' cases, each case with its own gains (clipped ones included);
  * Lift on the oracle through the environment API: "variable_kp" with kp = 150 in every action, and "variable" with kp = 150 and
    a damping ratio of 1, reproduce the fixed-mode trajectory bit for bit."""
import numpy as np
import pytest
import torch

from tests import controller_ref as ref
from tests import impedance_ref as imp
from tests.test_cpu_controllers import MODELS, _gate, from_oracle, oracle_inputs, to_oracle
from tests.util import lift_states, load

KINDS = {1: "OSC_POSE", 5: "OSC_POSITION", 3: "JOINT_POSITION"}
# Panda (7 joints): action_dim per kind and mode
ACTION_DIM = {(1, "fixed"): 7, (1, "variable"): 19, (1, "variable_kp"): 13,
              (5, "fixed"): 4, (5, "variable"): 16, (5, "variable_kp"): 10,
              (3, "fixed"): 8, (3, "variable"): 22, (3, "variable_kp"): 15}


def _cfg(kind, mode, robot="Panda", **part):
    from robosuite_b200.engine import CtrlCfg

    model = load(MODELS[robot])
    return model, ref.make_config(model, robot, kind, CtrlCfg, impedance_mode=mode, **part)


def _env(kind, mode, n=2, **part):
    import robosuite_b200 as suite
    from robosuite_b200 import controller_config as cc

    arm = cc.load_part_controller_config(KINDS[kind])
    arm.update(impedance_mode=mode, **part)
    return suite.make("Lift", robots="Panda", num_envs=n, seed=0, horizon=1000, sim_cls=imp.ImpedanceOracleSim,
                      controller_configs=cc.refactor_composite_controller_config(arm, "Panda", ["right"]))


@pytest.mark.parametrize("mode", ["fixed", "variable", "variable_kp"])
@pytest.mark.parametrize("kind", list(KINDS))
def test_resolve_action_dim_and_spec(kind, mode):
    env = _env(kind, mode)
    c = env._ctrl_cfg
    assert env.action_dim == c.action_dim == ACTION_DIM[(kind, mode)]
    low, high = env.action_spec
    assert low.shape == high.shape == (env.action_dim,)
    d = 7 if kind == 3 else 6
    od = {1: 6, 5: 3, 3: 7}[kind]
    gains = {"fixed": ([], []), "variable_kp": ([0.0] * d, [300.0] * d),
             "variable": ([0.0] * d + [0.0] * d, [10.0] * d + [300.0] * d)}[mode]
    assert list(low) == gains[0] + [-1.0] * od + [-1.0]
    assert list(high) == gains[1] + [1.0] * od + [1.0]
    # the gym wrapper's action space follows: a sample is a valid action
    from robosuite_b200.wrappers import BatchedGymWrapper

    w = BatchedGymWrapper(env)
    assert w.single_action_shape == (env.action_dim,)
    w.step(torch.as_tensor(np.stack([np.random.default_rng(0).uniform(low, high) for _ in range(2)])))
    env.close()


def test_resolve_broadcasts_limits():
    _, c = _cfg(1, "variable", kp_limits=[5, 200], damping_ratio_limits=[[0.1, 0.2, 0.3, 0.4, 0.5, 0.6], 4])
    assert list(c.kp_min)[:6] == [5.0] * 6 and list(c.kp_max)[:6] == [200.0] * 6
    assert list(c.damping_ratio_min)[:6] == [0.1, 0.2, 0.3, 0.4, 0.5, 0.6] and list(c.damping_ratio_max)[:6] == [4.0] * 6
    assert c.impedance_mode == imp.VARIABLE
    _, c = _cfg(5, "variable_kp", kp_limits=[[1, 2, 3, 4, 5, 6], 50])  # OSC_POSITION keeps a 6-dim kp
    assert list(c.kp_min)[:6] == [1.0, 2.0, 3.0, 4.0, 5.0, 6.0] and list(c.kp_max)[:6] == [50.0] * 6
    _, c = _cfg(3, "variable", kp_limits=[0, list(range(10, 17))])
    assert list(c.kp_max)[:7] == [float(v) for v in range(10, 17)] and list(c.kp_max)[7] == 0.0
    assert list(c.damping_ratio_max)[:7] == [10.0] * 7
    _, c = _cfg(1, "fixed")
    assert c.impedance_mode == imp.FIXED and c.action_dim == 7


def test_resolve_errors():
    from oracle.pyoracle import CtrlCfg as OCfg

    with pytest.raises(ValueError):
        _cfg(1, "sometimes")
    with pytest.raises(ValueError):  # a limit vector of the wrong length
        _cfg(3, "variable", kp_limits=[[0, 0, 0], 300])
    with pytest.raises(NotImplementedError):  # a struct without the appended fields cannot carry a variable mode
        model = load("Lift_Panda")
        ref.make_config(model, "Panda", 1, OCfg, impedance_mode="variable")
    for part in ({"input_type": "absolute"}, {"input_ref_frame": "world"}, {"interpolation": "linear"}):
        with pytest.raises(NotImplementedError) as ei:
            _cfg(1, "variable", **part)
        assert "fixed impedance" not in str(ei.value)
    with pytest.raises(NotImplementedError) as ei:
        _cfg(3, "variable_kp", qpos_limits=[-1, 1])
    assert "fixed impedance" not in str(ei.value)
    # the joint velocity and torque controllers have no impedance mode: the key is ignored, as the reference ignores it
    for kind in (2, 4):
        _, c = _cfg(kind, "variable")
        assert c.impedance_mode == imp.FIXED and c.action_dim == 8


def test_gains_against_hand_computed():
    _, c = _cfg(1, "variable")
    dr = [-1.0, 0.5, 12.0, 10.0, 0.0, 1.0]
    kp = [-5.0, 0.0, 150.0, 301.0, 300.0, 1e6]
    g = imp.gains_from_action(c, np.array(dr + kp + [0.0] * 7))
    assert list(g[:6]) == [0.0, 0.0, 150.0, 300.0, 300.0, 300.0]
    assert list(g[8:14]) == [0.0, 0.0, 2.0 * np.sqrt(150.0) * 10.0, 2.0 * np.sqrt(300.0) * 10.0, 0.0, 2.0 * np.sqrt(300.0)]
    assert not g[6:8].any() and not g[14:].any()
    _, c = _cfg(3, "variable_kp")
    g = imp.gains_from_action(c, np.array([-1.0, 0.0, 49.0, 300.0, 400.0, 25.0, 1.0] + [0.0] * 8))
    assert list(g[:7]) == [0.0, 0.0, 49.0, 300.0, 300.0, 25.0, 1.0]
    assert list(g[8:15]) == [0.0, 0.0, 14.0, 2.0 * np.sqrt(300.0), 2.0 * np.sqrt(300.0), 10.0, 2.0]
    # the configured gains in the action give the configured row exactly
    for kind in KINDS:
        for mode in ("variable", "variable_kp"):
            _, c = _cfg(kind, mode)
            row = imp.configured_gains(c)
            d = imp.gain_dim(c)
            dr = np.ones(d) if kind == 3 else np.array(list(c.damping_ratio)[:6])
            a = np.concatenate(([dr] if mode == "variable" else []) + [row[:d], np.zeros(c.action_dim - imp.delta_offset(c))])
            assert np.array_equal(imp.gains_from_action(c, a), row)


def case_gains(cfg, case, rng):
    """the gain part of a case's action: ordinary draws inside the limits; beyond them for "beyond_range" and "clip" (kp below 0
    and above kp_max, damping ratios beyond their limits); kp = 0 on one axis for "grip_saturated" """
    d = imp.gain_dim(cfg)
    kp, dr = rng.uniform(20.0, 280.0, d), rng.uniform(0.3, 2.0, d)
    if case in ("beyond_range", "clip"):
        kp = rng.choice([-40.0, 450.0], d)
        dr = rng.choice([-0.5, 14.0], d)
    elif case == "grip_saturated":
        kp[int(rng.integers(d))] = 0.0
    return np.concatenate(([dr] if int(cfg.impedance_mode) == imp.VARIABLE else []) + [kp])


def case_action(cfg, case, rng):
    """a case's variable-mode action: its gains, then controller_ref's delta and gripper action for the case"""
    delta = ref.case_action(ref_view(cfg), case, rng)
    return np.concatenate([case_gains(cfg, case, rng), delta])


def ref_view(cfg):
    return imp.fixed_view(cfg, imp.configured_gains(cfg))


VCONFIGS = [(robot, kind, mode) for robot in ("Panda", "Sawyer") for kind in KINDS for mode in ("variable", "variable_kp")]


def vconfig_id(c):
    return "%s-%s-%s" % (c[0], KINDS[c[1]], c[2])


@pytest.mark.parametrize("conf", VCONFIGS, ids=vconfig_id)
def test_restatement_matches_oracle_controller(conf):
    """test_cpu_controllers' case set with per-case gains: the oracle's controller runs on the delta part with the gains set in its
    configuration (what ImpedanceOracleSim does), the restatement from the whole action"""
    from oracle.pyoracle import CtrlCfg as OCfg
    from oracle.pyoracle import Oracle
    from robosuite_b200.mjcf.compiler import pack_model

    robot, kind, mode = conf
    model, cfg = _cfg(kind, mode, robot)
    o = Oracle(pack_model(model))
    oc = OCfg()
    for name, _ in OCfg._fields_:
        setattr(oc, name, getattr(cfg, name))
    oc.action_dim = cfg.action_dim - imp.delta_offset(cfg)
    o.ctrl_setup(oc)
    rng = np.random.default_rng(100 + kind + 7 * (mode == "variable") + 13 * (robot == "Sawyer"))
    acts = ref.controlled_actuators(cfg)
    d = imp.gain_dim(cfg)
    lim = {f: np.array(list(getattr(cfg, f))[:d]) for f in ("damping_ratio_min", "damping_ratio_max")}
    clipped = 0
    for case in ref.CASES:
        if robot != "Panda" and case in ref.PANDA_ONLY:
            continue
        o.reset_data()
        if robot == "Panda":
            o.qpos[:] = lift_states(model, 1, seed=int(rng.integers(1 << 30)))[0][0]
        qa, va = ref.case_arm(robot, case, rng)
        o.qpos[[cfg.arm_qpos[k] for k in range(7)]] = qa
        o.qvel[[cfg.arm_dof[k] for k in range(7)]] = va
        o.forward()
        st = ref.case_state(model, ref_view(cfg), case, rng, o.site_xpos, o.site_xmat, o.qpos)
        to_oracle(st, o.ctrl_state)
        action = case_action(cfg, case, rng)
        gain = imp.configured_gains(cfg)
        new = imp.gains_from_action(cfg, action)
        clipped += int(not np.array_equal(new[:d], action[imp.delta_offset(cfg) - d:imp.delta_offset(cfg)]))
        # the oracle's configuration carries the gains: OSC kd = 2 sqrt(kp) dr, joint position jv_kp / jv_kd
        if kind == 3:
            oc.jv_kp[:d], oc.jv_kd[:d] = list(new[:d]), list(new[8:8 + d])
        else:
            oc.kp[:6] = list(new[:6])
            oc.damping_ratio[:6] = list(np.clip(action[:6], lim["damping_ratio_min"], lim["damping_ratio_max"])
                                         if mode == "variable" else np.ones(6))
        gate = _gate(case, cfg)
        for sub in range(4):
            a = action if sub == 0 else None
            o.step1()
            inp = oracle_inputs(o)
            o.ctrl_run(None if a is None else a[imp.delta_offset(cfg):])
            r = imp.run(model, cfg, inp, st, gain, a, goal_ori=o.ctrl_state.goal_ori)
            assert np.array_equal(r["gain"], new), (case, sub)
            tau = np.array(o.ctrl_state.torques[:cfg.n_arm])
            assert np.isfinite(r["torque"]).all() and np.isfinite(tau).all(), (case, sub)
            err = np.abs(r["torque"] - tau).max() / max(1.0, np.abs(tau).max())
            assert err < gate, (case, sub, err)
            assert np.allclose(r["ctrl"][acts], o.ctrl[acts], rtol=0, atol=gate * max(1.0, np.abs(tau).max())), (case, sub)
            ost = from_oracle(o.ctrl_state)
            for k in ("goal_pos", "grip"):
                assert np.allclose(r["state"][k], ost[k], rtol=0, atol=1e-12), (case, sub, k)
            r["state"]["goal_ori"][:] = ost["goal_ori"]
            if kind == 3:
                assert np.allclose(r["state"]["jv"][:8], ost["jv"][:8], rtol=0, atol=1e-12), (case, sub)
            st, gain = r["state"], r["gain"]
            o.step2()
    assert clipped > 0  # some case's gains were clipped


@pytest.mark.parametrize("mode", ["variable", "variable_kp"])
def test_lift_with_configured_gains_reproduces_fixed_mode(mode):
    """Lift / Panda, OSC_POSE on the oracle through the environment API: the configured kp = 150 (and damping ratio 1) in every
    action reproduce the fixed-mode trajectory bit for bit, through a reset"""
    rng = np.random.default_rng(3)
    fixed, var = _env(1, "fixed"), _env(1, mode)
    d = imp.delta_offset(var._ctrl_cfg)
    gains = [1.0] * 6 + [150.0] * 6 if mode == "variable" else [150.0] * 6
    assert len(gains) == d
    for env in (fixed, var):
        env.reset()
    for t in range(6):
        a = rng.uniform(-1, 1, (2, 7))
        fixed.step(torch.as_tensor(a))
        var.step(torch.as_tensor(np.concatenate([np.tile(gains, (2, 1)), a], axis=1)))
        assert torch.equal(fixed.sim.qpos, var.sim.qpos) and torch.equal(fixed.sim.qvel, var.sim.qvel), t
        assert torch.equal(fixed.sim.ctrl, var.sim.ctrl), t
        if t == 2:
            for env in (fixed, var):
                env.reset()
    assert np.array_equal(var.sim.ctrl_gain.numpy(), np.tile(imp.configured_gains(var._ctrl_cfg), (2, 1)))
    fixed.close()
    var.close()
