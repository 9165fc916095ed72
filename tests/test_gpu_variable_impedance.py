"""GPU: variable impedance (impedance_mode "variable" / "variable_kp") of OSC_POSE, OSC_POSITION and JOINT_POSITION on the device.

  * Against the restatement (tests/impedance_ref.py over tests/controller_ref.py), as test_gpu_controllers does it: 37 environments
    in 3 groups, each with its own case, gains (clipped ones and kp = 0 included, test_cpu_variable_impedance.case_gains) and
    action, every placement, f64 and f32, the policy substep and a later one; ctrl_torque, ctrl, the controller state and
    ctrl_gain are compared under that file's gates.  The gains themselves are fp64 arithmetic on the action in both precisions
    and must match bit for bit.
  * The configured gains in the action give fixed mode's bits in every placement.
  * The three schedules agree bit for bit with per-environment gains, through a masked reset, with a small tail tier.
  * Snapshot, restore and clone carry the gains; a fixed-mode handle has the section table and signature it always had.
  * Lift / Panda with OSC_POSE "variable" in lockstep with the oracle through the environment API.
  * Joint position with "variable" (22 action entries) runs in every placement.
  * b2s_ctrl_impedance rejects what it must."""
import numpy as np
import pytest

from tests import controller_ref as ref
from tests import impedance_ref as imp
from tests.schedules import switches
from tests.test_cpu_controllers import MODELS, NEAR_GATES
from tests.test_cpu_variable_impedance import KINDS, VCONFIGS, case_action, ref_view, vconfig_id
from tests.test_gpu_controllers import F32_GATES, ILL, PLACEMENTS, STATE_ARRAYS, _cases, _inputs, _np, _read_state
from tests.util import lift_states, load

pytestmark = pytest.mark.gpu

N = 37


def _setup(robot, kind, mode, precision):
    import torch

    from robosuite_b200.engine import BatchedSim, CtrlCfg

    model = load(MODELS[robot])
    sim = BatchedSim(model, N, precision=precision)
    cfg = ref.make_config(model, robot, kind, CtrlCfg, impedance_mode=mode)
    sim.ctrl_config(cfg)
    rng = np.random.default_rng(1000 * kind + 7 * (mode == "variable") + (robot == "Sawyer"))
    cases = [_cases(robot)[e % len(_cases(robot))] for e in range(N)]
    q = lift_states(model, N, seed=5)[0] if robot == "Panda" else np.tile(model.qpos0, (N, 1))
    v = np.zeros((N, model.nv))
    arm_q = [cfg.arm_qpos[k] for k in range(cfg.n_arm)]
    arm_v = [cfg.arm_dof[k] for k in range(cfg.n_arm)]
    for e, case in enumerate(cases):
        q[e, arm_q], v[e, arm_v] = ref.case_arm(robot, case, rng)
    dt = sim.dtype
    sim.qpos.copy_(torch.as_tensor(q, dtype=dt))
    sim.qvel.copy_(torch.as_tensor(v, dtype=dt))
    sim.forward()
    sim.ctrl_reset()
    torch.cuda.synchronize()
    assert np.array_equal(_np(sim.array("ctrl_gain")), np.tile(imp.configured_gains(cfg), (N, 1)))
    sxp, sxm, qp = _np(sim.site_xpos).reshape(N, -1, 3), _np(sim.site_xmat).reshape(N, -1, 9), _np(sim.qpos)
    states = [ref.case_state(model, ref_view(cfg), case, rng, sxp[e], sxm[e], qp[e]) for e, case in enumerate(cases)]
    for k, a in STATE_ARRAYS.items():
        sim.array(a).copy_(torch.as_tensor(np.stack([s[k] for s in states]), dtype=dt))
    d = imp.gain_dim(cfg)
    g0 = np.zeros((N, 16))  # each environment starts from gains of its own (a later substep reads the policy substep's)
    g0[:, :d], g0[:, 8:8 + d] = rng.uniform(10, 250, (N, d)), rng.uniform(1, 40, (N, d))
    sim.array("ctrl_gain").copy_(torch.as_tensor(g0))
    actions = np.stack([case_action(cfg, case, rng) for case in cases])
    sim.set_export(False)
    sim.set_step1_export(True)
    torch.cuda.synchronize()
    return sim, cfg, cases, torch.as_tensor(actions, dtype=dt, device=sim.torch_device).contiguous()


def _compare(sim, cfg, cases, q0, v0, st0, g0, actions, policy, precision, worst):
    """test_gpu_controllers._compare with the gains: the last substep of the call just made against the restatement"""
    model = sim.model
    tau_d, ctrl_d, st_d = _np(sim.ctrl_torque)[:, :cfg.n_arm], _np(sim.ctrl), _read_state(sim)
    gain_d = _np(sim.array("ctrl_gain"))
    warn = sim.warn.cpu().numpy()
    acts = ref.controlled_actuators(cfg)
    arm_u = [cfg.arm_act[k] for k in range(cfg.n_arm)]
    lo, hi = model.actuator_ctrlrange[arm_u, 0], model.actuator_ctrlrange[arm_u, 1]
    f64 = precision == "f64"
    for e, case in enumerate(cases):
        tag = (e, case, "policy" if policy else "later")
        inp = _inputs(sim, e)
        inp["qpos"], inp["qvel"] = q0[e], v0[e]
        st = {k: v[e] for k, v in st0.items()}
        r = imp.run(model, cfg, inp, st, g0[e], actions[e] if policy else None, goal_ori=st_d["goal_ori"][e])
        assert np.array_equal(gain_d[e], r["gain"]), tag + (gain_d[e], r["gain"])
        assert warn[e] == 0, tag + (int(warn[e]), tau_d[e])
        assert np.isfinite(tau_d[e]).all() and np.isfinite(ctrl_d[e, acts]).all(), tag
        assert np.array_equal(ctrl_d[e, arm_u], np.clip(tau_d[e], lo, hi)), tag
        scale = max(1.0, np.abs(r["torque"]).max())
        err = np.abs(tau_d[e] - r["torque"]).max() / scale
        ill = cfg.kind in (1, 5) and case in ILL
        worst[case] = max(worst.get(case, 0.0), err)
        if f64:
            gate = NEAR_GATES.get(case, 1e-12) if cfg.kind in (1, 5) else 1e-12
        else:
            gate = F32_GATES["ill" if ill else "torque"]
        assert err < gate, tag + (err, gate)
        assert np.allclose(ctrl_d[e, acts], r["ctrl"][acts], rtol=0, atol=gate * scale), tag
        sg = 1e-12 if f64 else F32_GATES["state"]
        for k in ("goal_pos", "grip", "initial_joint"):
            assert np.allclose(st_d[k][e], r["state"][k], rtol=sg, atol=sg), tag + (k,)
        assert np.allclose(st_d["goal_ori"][e], r["state"]["goal_ori"], rtol=0, atol=5e-7 if policy else sg), tag
        if cfg.kind == 3:
            assert np.allclose(st_d["jv"][e][:8], r["state"]["jv"][:8], rtol=sg, atol=sg), tag


@pytest.mark.parametrize("placement", list(PLACEMENTS))
@pytest.mark.parametrize("precision", ["f64", "f32"])
@pytest.mark.parametrize("conf", VCONFIGS, ids=vconfig_id)
def test_device_gains_match_restatement(conf, precision, placement):
    import torch

    robot, kind, mode = conf
    mode_id, split = PLACEMENTS[placement]
    worst = {}
    with switches(ctrl_split=split, groups=3):
        sim, cfg, cases, actions = _setup(robot, kind, mode, precision)
        sim.set_mode(mode_id)
        acts_np = _np(actions)
        q0, v0, st0, g0 = _np(sim.qpos), _np(sim.qvel), _read_state(sim), _np(sim.array("ctrl_gain"))
        snap = sim.snapshot()
        sim.env_step(actions, 1)
        torch.cuda.synchronize()
        _compare(sim, cfg, cases, q0, v0, st0, g0, acts_np, True, precision, worst)
        sim.restore(snap)
        sim.env_step(actions, 2)
        torch.cuda.synchronize()
        q2, v2, st2, g2 = _np(sim.qpos), _np(sim.qvel), _read_state(sim), _np(sim.array("ctrl_gain"))
        sim.restore(snap)
        sim.env_step(actions, 3)
        torch.cuda.synchronize()
        _compare(sim, cfg, cases, q2, v2, st2, g2, acts_np, False, precision, worst)
        sim.close()
    print("%s %s %s worst torque rel err: %s" % (vconfig_id(conf), precision, placement, {k: "%.2g" % v for k, v in worst.items()}))


def _lift_pair(kind, mode, precision, n=16):
    """a fixed-mode and a variable-mode Lift / Panda handle of `kind` from the same states"""
    import torch

    from robosuite_b200.engine import BatchedSim, CtrlCfg

    model = load("Lift_Panda")
    q, _ = lift_states(model, n, seed=21)
    out = []
    for m in ("fixed", mode):
        sim = BatchedSim(model, n, precision=precision)
        cfg = ref.make_config(model, "Panda", kind, CtrlCfg, impedance_mode=m)
        sim.ctrl_config(cfg)
        sim.set_export(False)
        sim.qpos.copy_(torch.as_tensor(q, dtype=sim.dtype))
        sim.forward()
        sim.ctrl_reset()
        out.append((sim, cfg))
    return out


@pytest.mark.parametrize("placement", list(PLACEMENTS))
@pytest.mark.parametrize("mode", ["variable", "variable_kp"])
@pytest.mark.parametrize("kind", list(KINDS))
def test_configured_gains_give_fixed_bits(kind, mode, placement):
    import torch

    mode_id, split = PLACEMENTS[placement]
    rng = np.random.default_rng(kind)
    with switches(ctrl_split=split, groups=3):
        (fs, fcfg), (vs, vcfg) = _lift_pair(kind, mode, "f32")
        for s in (fs, vs):
            s.set_mode(mode_id)
        row = imp.configured_gains(vcfg)
        for t in range(4):
            a = rng.uniform(-1, 1, (fs.n_env, fcfg.action_dim))
            va = np.stack([imp.gain_action(vcfg, row, a[e]) for e in range(fs.n_env)])
            assert np.array_equal(np.stack([imp.gains_from_action(vcfg, x) for x in va]), np.tile(row, (fs.n_env, 1)))
            fs.env_step(torch.as_tensor(a, dtype=fs.dtype, device=fs.torch_device).contiguous(), 5)
            vs.env_step(torch.as_tensor(va, dtype=vs.dtype, device=vs.torch_device).contiguous(), 5)
        torch.cuda.synchronize()
        for f in ("qpos", "qvel", "ctrl", "ctrl_torque"):
            assert torch.equal(getattr(fs, f), getattr(vs, f)), f
        fs.close()
        vs.close()


def _gain_actions(cfg, calls, n, seed):
    """per-environment gains inside and beyond the limits, then lift_actions-like deltas with the gripper closing"""
    rng = np.random.default_rng(seed)
    d = imp.gain_dim(cfg)
    out = []
    for _ in range(calls):
        kp = rng.uniform(-30, 330, (n, d))
        parts = [kp, rng.uniform(-1, 1, (n, cfg.action_dim - imp.delta_offset(cfg)))]
        if int(cfg.impedance_mode) == imp.VARIABLE:
            parts.insert(0, rng.uniform(-0.5, 3.0, (n, d)))
        a = np.concatenate(parts, axis=1)
        a[:, -1] = 1.0
        out.append(a)
    return np.stack(out)


@pytest.mark.parametrize("mode", ["variable", "variable_kp"])
@pytest.mark.parametrize("kind", [1, 3])
def test_schedules_agree_with_per_environment_gains(kind, mode):
    """fused kernel, pipeline and unit queue bit-identical with per-environment gains, through a masked reset, small tail tier"""
    import torch

    from robosuite_b200.engine import BatchedSim, CtrlCfg

    model = load("Lift_Panda")
    n = 16
    q, _ = lift_states(model, n, seed=21)
    res = []
    for mode_id in (0, 1, 2):
        with switches(gjk_cache=False, ctrl_split=False, groups=3):
            sim = BatchedSim(model, n, precision="f32", tier_small=(4, 24))
            cfg = ref.make_config(model, "Panda", kind, CtrlCfg, impedance_mode=mode)
            sim.ctrl_config(cfg)
            sim.set_export(False)
            sim.set_mode(mode_id)
            sim.qpos.copy_(torch.as_tensor(q, dtype=sim.dtype))
            sim.forward()
            sim.ctrl_reset()
            acts = _gain_actions(cfg, 8, n, seed=kind)
            mask = torch.zeros(n, dtype=torch.uint8, device=sim.torch_device)
            mask[::3] = 1
            for t in range(8):
                if t == 4:
                    sim.reset_envs(mask, torch.as_tensor(q, dtype=sim.dtype, device=sim.torch_device))
                    torch.cuda.synchronize()
                    g = _np(sim.array("ctrl_gain"))
                    assert np.array_equal(g[::3], np.tile(imp.configured_gains(cfg), (len(g[::3]), 1)))
                sim.env_step(torch.as_tensor(acts[t], dtype=sim.dtype, device=sim.torch_device).contiguous(), 10)
            torch.cuda.synchronize()
            res.append(tuple(_np(getattr(sim, f)) if f != "ctrl_gain" else _np(sim.array(f)) for f in ("qpos", "qvel", "ctrl", "ctrl_gain")))
            assert np.isfinite(res[-1][0]).all() and int(sim.warn.abs().max()) == 0
            sim.close()
    for other in res[1:]:
        for a, b in zip(res[0], other):
            assert np.array_equal(a, b)


def test_snapshots_carry_the_gains():
    import torch

    from robosuite_b200.engine import BatchedSim, CtrlCfg

    model = load("Lift_Panda")
    n = 8
    q, _ = lift_states(model, n, seed=4)
    fixed = BatchedSim(model, n, precision="f32")
    fixed.ctrl_config(ref.make_config(model, "Panda", 1, CtrlCfg))
    rb0, sig0, secs0 = fixed.snapshot_layout()
    assert "ctrl_gain" not in [s[0] for s in secs0]
    sim = BatchedSim(model, n, precision="f32")
    cfg = ref.make_config(model, "Panda", 1, CtrlCfg, impedance_mode="variable")
    sim.ctrl_config(cfg)
    rb, sig, secs = sim.snapshot_layout()
    names = [s[0] for s in secs]
    assert "ctrl_gain" in names and sig != sig0 and rb > rb0
    sim.set_export(False)
    sim.set_mode(1)
    sim.qpos.copy_(torch.as_tensor(q, dtype=sim.dtype))
    sim.forward()
    sim.ctrl_reset()
    acts = _gain_actions(cfg, 4, n, seed=9)
    step = lambda t: sim.env_step(torch.as_tensor(acts[t], dtype=sim.dtype, device=sim.torch_device).contiguous(), 10)
    step(0)
    snap = sim.snapshot()
    g_snap = _np(sim.array("ctrl_gain"))
    step(1)
    # the later substeps of a call read the gains of its policy substep: a restored row must bring them back
    sim.restore(snap)
    assert np.array_equal(_np(sim.array("ctrl_gain")), g_snap)
    # clone: environment e takes environment src[e]'s gains with the rest of its state
    src = [3] * n
    sim.clone_envs(src)
    torch.cuda.synchronize()
    assert np.array_equal(_np(sim.array("ctrl_gain")), np.tile(g_snap[3], (n, 1)))
    # variable -> variable_kp changes the signature; back to fixed gives the fixed table and signature again
    sim.ctrl_config(ref.make_config(model, "Panda", 1, CtrlCfg, impedance_mode="variable_kp"))
    assert sim.snapshot_layout()[1] not in (sig, sig0)
    sim.ctrl_config(ref.make_config(model, "Panda", 1, CtrlCfg))
    rb1, sig1, secs1 = sim.snapshot_layout()
    assert (rb1, sig1) == (rb0, sig0) and [s[0] for s in secs1] == [s[0] for s in secs0]
    sim.close()
    fixed.close()


def test_lift_osc_variable_matches_oracle():
    """Lift / Panda, OSC_POSE "variable", f64 pipeline against ImpedanceOracleSim through the environment API, with actions drawn
    from action_spec (gains across their whole range); the tolerances of test_gpu_env's environment comparisons"""
    import torch

    import robosuite_b200 as suite
    from robosuite_b200 import controller_config as cc

    arm = cc.load_part_controller_config("OSC_POSE")
    arm["impedance_mode"] = "variable"
    ctrl = cc.refactor_composite_controller_config(arm, "Panda", ["right"])
    n = 4
    dev = suite.make("Lift", robots="Panda", num_envs=n, seed=0, horizon=1000, controller_configs=ctrl, precision="f64")
    orc = suite.make("Lift", robots="Panda", num_envs=n, seed=0, horizon=1000, controller_configs=ctrl, sim_cls=imp.ImpedanceOracleSim)
    assert dev.action_dim == orc.action_dim == 19
    low, high = dev.action_spec
    dev.reset()  # the device's placement draws, replayed on the oracle
    q0 = dev.sim.qpos.cpu().numpy()
    dev.reset_to(torch.as_tensor(q0))
    orc.reset_to(q0)
    rng = np.random.default_rng(5)
    for t in range(10):
        a = rng.uniform(low, high, (n, dev.action_dim))
        dev.step(torch.as_tensor(a, dtype=dev.dtype, device=dev.device))
        orc.step(torch.as_tensor(a))
        torch.cuda.synchronize()
        dq = np.abs(dev.sim.qpos.cpu().numpy() - orc.sim.qpos.numpy()).max()
        assert dq < 1e-6, (t, dq)
        assert np.array_equal(_np(dev.sim.array("ctrl_gain")), orc.sim.ctrl_gain.numpy()), t
    dev.close()
    orc.close()


@pytest.mark.parametrize("placement", list(PLACEMENTS))
def test_largest_action_runs_everywhere(placement):
    """joint position with "variable": 3 x 7 + 1 = 22 action entries, past the previous cap of 16"""
    import torch

    mode_id, split = PLACEMENTS[placement]
    with switches(ctrl_split=split, groups=3):
        (fs, _), (vs, vcfg) = _lift_pair(3, "variable", "f32", n=8)
        fs.close()
        assert vcfg.action_dim == 22
        vs.set_mode(mode_id)
        acts = _gain_actions(vcfg, 3, vs.n_env, seed=1)
        for a in acts:
            vs.env_step(torch.as_tensor(a, dtype=vs.dtype, device=vs.torch_device).contiguous(), 5)
        torch.cuda.synchronize()
        g = _np(vs.array("ctrl_gain"))
        assert np.array_equal(g, np.stack([imp.gains_from_action(vcfg, x) for x in acts[-1].astype(np.float32).astype(np.float64)]))
        assert np.isfinite(_np(vs.qpos)).all() and int(vs.warn.abs().max()) == 0
        vs.close()


def test_ctrl_config_rejects_bad_impedance():
    """b2s_ctrl_impedance: an unknown mode, a variable mode with another kind, bad limits and a wrong action_dim are B2S_ERR_ARG"""
    from robosuite_b200.engine import B2SError, BatchedSim, CtrlCfg

    model = load("Lift_Panda")
    sim = BatchedSim(model, 4, precision="f32")
    good = ref.make_config(model, "Panda", 1, CtrlCfg, impedance_mode="variable")
    sim.ctrl_config(good)

    def bad(kind=1, **fields):
        c = ref.make_config(model, "Panda", kind, CtrlCfg, impedance_mode="variable" if kind in (1, 3, 5) else "fixed")
        for f, v in fields.items():
            if isinstance(v, tuple):
                getattr(c, f)[v[0]] = v[1]
            else:
                setattr(c, f, v)
        with pytest.raises(B2SError):
            sim.ctrl_config(c)

    bad(impedance_mode=3)
    bad(2, impedance_mode=1)
    bad(4, impedance_mode=2)
    bad(kp_min=(2, -1.0))
    bad(kp_max=(5, float("inf")))
    bad(damping_ratio_min=(0, float("nan")))
    bad(kp_min=(1, 301.0))
    bad(damping_ratio_min=(3, 11.0))
    bad(action_dim=13)
    bad(3, action_dim=21)
    sim.close()
