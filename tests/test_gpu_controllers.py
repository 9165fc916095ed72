"""GPU: every controller placement against the fp64 restatement of the reference's controllers (tests/controller_ref.py), substep
by substep.

Each test writes qpos, qvel and the controller state arrays of 37 environments (not a multiple of 32, in 3 pipeline groups), each
with its own case of controller_ref.CASES (ordinary, actions beyond the input range with a gripper action of 0, a saturated gripper
integrator, torques beyond ctrlrange, and on the Panda the singular pose and three poses near it) and its own action.  It turns on
the step-1 export and compares ctrl_torque, ctrl and the new controller state with the restatement evaluated on the device's own
exported inputs (poses, cdof, qM, qfrc_bias) cast to fp64, so the controller is judged apart from the dynamics' rounding:
  * the policy substep: env_step(a, 1);
  * a later substep (no new goal): env_step(a, 2) and env_step(a, 3) from the same snapshot; the first supplies qpos, qvel and the
    controller state at the start of substep 3, the second the poses of substep 3.
Placements: the fused kernel (mode 0), the pipeline with its thread-per-environment OSC kernel (mode 1) and with the controller
inside the tail (B2S_CTRL_SPLIT=0), and the unit queue (mode 2).

Gates (relative to the largest torque, or 1 N m):
  * f64: 1e-12, and at and near the singular pose the conditioning gates of test_cpu_controllers.NEAR_GATES.  The orientation goal
    of a policy substep is formed in float32 as the reference does, compared at float32 precision, and the torques are judged on the
    device's goal (controller_ref.run_given_goal).
  * f32: F32_GATES, about 5x the worst measured on an H100 80GB HBM3 at a 700 W power limit.  At the singular and near-singular
    Panda poses the fp32 Jacobian leaves the smallest eigenvalue of J M^-1 J^T anywhere from below pinv's cut-off to ~1e-7 of the
    largest, so the OSC torques there are decided by fp32 rounding: those cases are gated on what the reference determines (finite
    torques, no warn bit, ctrl the clip of ctrl_torque, the goals and gripper state) and on the loosest conditioning gate of the
    f64 comparison; their measured spread was 7.8e-5 (coupled OSC_POSE, near_1e-5, every placement).

Measured worst relative torque errors on that card, f64, over every placement: 1.4e-14 away from the singularity (4.6e-16 for the
joint controllers); singular 7.3e-11, near_1e-3 1.5e-10, near_1e-5 1.3e-6, near_1e-7 6.4e-3.  f32: 2.9e-6 for the OSC and 2.3e-6
for the joint controllers.  Every test prints its worst per case."""
import numpy as np
import pytest

from tests import controller_ref as ref
from tests.schedules import switches
from tests.test_cpu_controllers import CONFIGS, MODELS, NEAR_GATES, config_id
from tests.util import lift_states, load

pytestmark = pytest.mark.gpu

N = 37
PLACEMENTS = {"fused": (0, True), "pipeline": (1, True), "pipeline_unsplit": (1, False), "unit_queue": (2, True)}
# f32 gates: relative torque (worst measured 2.9e-6, Sawyer OSC_POSITION), relative torque at the ill-conditioned poses (the
# loosest conditioning gate of the f64 comparison; measured spread below) and the controller state (goals, gripper and
# joint-controller state; worst measured 5.3e-8)
F32_GATES = {"torque": 1.5e-5, "ill": NEAR_GATES["near_1e-7"], "state": 3e-7}
ILL = ref.PANDA_ONLY  # the cases whose fp32 OSC torques rounding decides


def _cases(robot):
    return [c for c in ref.CASES if robot == "Panda" or c not in ref.PANDA_ONLY]


def _np(t):
    return t.detach().cpu().numpy().astype(np.float64)


def _inputs(sim, e):
    return dict(qpos=None, qvel=None, site_xpos=_np(sim.site_xpos[e]).reshape(-1, 3), site_xmat=_np(sim.site_xmat[e]).reshape(-1, 9),
                cdof=_np(sim.cdof[e]).reshape(-1, 6), qM=_np(sim.qM[e]).reshape(sim.model.nv, sim.model.nv),
                qfrc_bias=_np(sim.qfrc_bias[e]))


STATE_ARRAYS = {"goal_pos": "ctrl_goal_pos", "goal_ori": "ctrl_goal_ori", "initial_joint": "ctrl_initial_joint",
                "grip": "ctrl_grip_state", "jv": "ctrl_jv_state"}


def _read_state(sim):
    return {k: _np(sim.array(a)) for k, a in STATE_ARRAYS.items()}


def _setup(robot, kind, over, precision, placement):
    import torch

    from robosuite_b200.engine import BatchedSim, CtrlCfg

    model = load(MODELS[robot])
    mode, split = PLACEMENTS[placement]
    sim = BatchedSim(model, N, precision=precision)
    cfg = ref.make_config(model, robot, kind, CtrlCfg, **over)
    sim.ctrl_config(cfg)
    sim.set_mode(mode)
    rng = np.random.default_rng(1000 * kind + 7 * len(over) + (robot == "Sawyer"))
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
    sxp, sxm, qp = _np(sim.site_xpos).reshape(N, -1, 3), _np(sim.site_xmat).reshape(N, -1, 9), _np(sim.qpos)
    states = [ref.case_state(model, cfg, case, rng, sxp[e], sxm[e], qp[e]) for e, case in enumerate(cases)]
    for k, a in STATE_ARRAYS.items():
        sim.array(a).copy_(torch.as_tensor(np.stack([s[k] for s in states]), dtype=dt))
    actions = np.stack([ref.case_action(cfg, case, rng) for case in cases])
    sim.set_export(False)
    sim.set_step1_export(True)
    torch.cuda.synchronize()
    return sim, cfg, cases, torch.as_tensor(actions, dtype=dt, device=sim.torch_device).contiguous()


def _compare(sim, cfg, cases, q0, v0, st0, actions, policy, precision, worst):
    """the last substep of the call just made against the restatement; q0, v0, st0: qpos, qvel and controller state at its start"""
    model = sim.model
    tau_d = _np(sim.ctrl_torque)[:, :cfg.n_arm]
    ctrl_d = _np(sim.ctrl)
    st_d = _read_state(sim)
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
        a = actions[e] if policy else None
        r = ref.run_given_goal(model, cfg, inp, st, a, st_d["goal_ori"][e])
        assert warn[e] == 0, tag + (int(warn[e]), tau_d[e])
        assert np.isfinite(tau_d[e]).all() and np.isfinite(ctrl_d[e, acts]).all(), tag
        # ctrl of the arm is the clip of the device's own torques
        assert np.allclose(ctrl_d[e, arm_u], np.clip(tau_d[e], lo, hi), rtol=0, atol=0), tag
        scale = max(1.0, np.abs(r["torque"]).max())
        err = np.abs(tau_d[e] - r["torque"]).max() / scale
        ill = cfg.kind in (1, 5) and case in ILL
        key = (case, "policy" if policy else "later")
        worst[key] = max(worst.get(key, 0.0), err)
        if f64:
            gate = NEAR_GATES.get(case, 1e-12) if cfg.kind in (1, 5) else 1e-12
        else:
            gate = F32_GATES["ill" if ill else "torque"]
        assert err < gate, tag + (err, gate)
        assert np.allclose(ctrl_d[e, acts], r["ctrl"][acts], rtol=0, atol=gate * scale), tag
        sg = 1e-12 if f64 else F32_GATES["state"]
        serr = max(np.abs(st_d[k][e] - r["state"][k]).max() / max(1.0, np.abs(r["state"][k]).max()) for k in ("goal_pos", "grip", "jv"))
        worst["state"] = max(worst.get("state", 0.0), serr)
        for k in ("goal_pos", "grip", "initial_joint"):
            assert np.allclose(st_d[k][e], r["state"][k], rtol=sg, atol=sg), tag + (k,)
        assert np.allclose(st_d["goal_ori"][e], r["state"]["goal_ori"], rtol=0, atol=5e-7 if policy else sg), tag
        jv_d, jv_r = st_d["jv"][e], r["state"]["jv"]
        if cfg.kind == 2:
            assert np.array_equal(jv_d[64:67], jv_r[64:67]), tag + (jv_d[64:67], jv_r[64:67])
            assert np.allclose(jv_d[:64], jv_r[:64], rtol=sg, atol=sg * max(1.0, np.abs(jv_r[:64]).max())), tag
        elif cfg.kind in (3, 4):
            assert np.allclose(jv_d[:8], jv_r[:8], rtol=sg, atol=sg), tag


@pytest.mark.parametrize("placement", list(PLACEMENTS))
@pytest.mark.parametrize("precision", ["f64", "f32"])
@pytest.mark.parametrize("conf", CONFIGS, ids=config_id)
def test_device_controller_matches_restatement(conf, precision, placement):
    import torch

    robot, kind, over = conf
    mode, split = PLACEMENTS[placement]
    worst = {}
    with switches(ctrl_split=split, groups=3):
        sim, cfg, cases, actions = _setup(robot, kind, over, precision, placement)
        acts_np = _np(actions)
        q0, v0, st0 = _np(sim.qpos), _np(sim.qvel), _read_state(sim)
        snap = sim.snapshot()
        # the policy substep
        sim.env_step(actions, 1)
        torch.cuda.synchronize()
        _compare(sim, cfg, cases, q0, v0, st0, acts_np, True, precision, worst)
        # substep 3 of a call: its start from env_step(a, 2), its poses from env_step(a, 3)
        sim.restore(snap)
        sim.env_step(actions, 2)
        torch.cuda.synchronize()
        q2, v2, st2 = _np(sim.qpos), _np(sim.qvel), _read_state(sim)
        sim.restore(snap)
        sim.env_step(actions, 3)
        torch.cuda.synchronize()
        _compare(sim, cfg, cases, q2, v2, st2, acts_np, False, precision, worst)
        sim.close()
    print("%s %s %s worst torque rel err: %s" % (config_id(conf), precision, placement,
                                                 {"/".join(k) if isinstance(k, tuple) else k: "%.2g" % v for k, v in sorted(worst.items(), key=str)}))
