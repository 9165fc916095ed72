"""CPU: the fp64 restatement of the reference's controllers (tests/controller_ref.py) pinned to
  * the reference's own records: tests/golden/osc_golden.npz (OperationalSpaceController: torques, goals, ctrl) and
    tests/golden/jv_golden.npz (JointVelocityController: clipped torques, goal velocities, ctrl, saturation flags), replayed on the
    oracle's physics with the restatement writing ctrl;
  * the oracle's controller (oracle/o_ctrl.c) on the oracle's fp64 state, substep by substep, for every controller kind on the
    Panda and the Sawyer, coupled and uncoupled OSC, torque compensation off, velocity limits off, actions beyond the input range,
    a gripper action of exactly 0, a saturated gripper integrator, torques beyond ctrlrange, 8 consecutive substeps (the joint
    velocity controller's derivative ring wraps and its anti-windup flag toggles), the singular Panda pose and three poses near it.

Gates are at rounding (1e-12 relative to the largest torque, or 1 N m) away from the singularity.  At and near it, pinv keeps
eigenvalues of J M^-1 J^T down to 1e-15 of the largest, so lambda_full carries their inverse and the torques are only as well
determined as rounding times that condition number (NEAR_GATES).  The orientation goal of a policy substep is formed in float32 as
the reference does; it is compared at float32 precision and the torques are judged on the oracle's goal (controller_ref.run_given_goal)."""
import os

import numpy as np
import pytest

from tests import controller_ref as ref
from tests.util import ROOT, dedegenerate_sawyer, lift_states, load

MODELS = {"Panda": "Lift_Panda", "Sawyer": "Lift_Sawyer"}
# (robot, kind, part-config overrides): every kind on both arms; OSC coupled and uncoupled; JV with and without velocity limits;
# the joint controllers with torque compensation off
CONFIGS = [
    ("Panda", 1, {}), ("Panda", 1, {"uncouple_pos_ori": False}), ("Panda", 5, {}),
    ("Panda", 2, {}), ("Panda", 2, {"velocity_limits": None, "use_torque_compensation": False}),
    ("Panda", 3, {}), ("Panda", 3, {"use_torque_compensation": False}), ("Panda", 4, {}), ("Panda", 4, {"use_torque_compensation": False}),
    ("Sawyer", 1, {}), ("Sawyer", 1, {"uncouple_pos_ori": False}), ("Sawyer", 5, {}),
    ("Sawyer", 2, {}), ("Sawyer", 3, {}), ("Sawyer", 4, {"use_torque_compensation": False}),
]


def config_id(c):
    robot, kind, over = c
    return "-".join([robot, ref.KIND_NAMES[kind]] + ["%s=%s" % kv for kv in sorted(over.items())])


def oracle_inputs(o):
    return dict(qpos=o.qpos.copy(), qvel=o.qvel.copy(), site_xpos=o.site_xpos.copy(), site_xmat=o.site_xmat.copy(),
                cdof=o.cdof.copy(), qM=o.M.copy(), qfrc_bias=o.qfrc_bias.copy())


def from_oracle(st):
    jv = np.zeros(72)
    jv[:8], jv[8:16], jv[16:24] = st.jv_goal, st.jv_last_err, st.jv_summed
    jv[24:64] = np.array([list(r) for r in st.jv_derr]).reshape(40)
    jv[64], jv[65], jv[66] = st.jv_ptr, st.jv_size, st.jv_saturated
    return dict(goal_pos=np.array(st.goal_pos), goal_ori=np.array(st.goal_ori), initial_joint=np.array(st.initial_joint),
                grip=np.array(st.grip_action), jv=jv)


def to_oracle(d, st):
    st.goal_pos[:] = list(d["goal_pos"]); st.goal_ori[:] = list(d["goal_ori"])
    st.initial_joint[:] = list(d["initial_joint"]); st.grip_action[:] = list(d["grip"])
    jv = d["jv"]
    st.jv_goal[:], st.jv_last_err[:], st.jv_summed[:] = list(jv[:8]), list(jv[8:16]), list(jv[16:24])
    for r in range(5):
        st.jv_derr[r][:] = list(jv[24 + 8 * r:32 + 8 * r])
    st.jv_ptr, st.jv_size, st.jv_saturated = int(jv[64]), int(jv[65]), int(jv[66])


def _oracle(model, cfg):
    from oracle.pyoracle import Oracle
    from robosuite_b200.mjcf.compiler import pack_model

    o = Oracle(pack_model(model))
    o.ctrl_setup(cfg)
    return o


def test_restatement_jacobian_is_the_oracles():
    """the site Jacobian formed from cdof (the engine's convention) is mj_jacSite"""
    from oracle.pyoracle import CtrlCfg

    for robot in ("Panda", "Sawyer"):
        model = load(MODELS[robot])
        cfg = ref.make_config(model, robot, 1, CtrlCfg)
        o = _oracle(model, cfg)
        o.reset_data()
        o.qpos[:7] = ref.ARM_HOME[robot] + 0.3
        o.step1()
        for site in (cfg.eef_site, cfg.base_site):
            jp, jr = o.jac(o.site_xpos[site], int(model.site_bodyid[site]))
            J = ref.site_jacobian(model, o.cdof, site, o.site_xpos[site])
            assert np.abs(J - np.vstack([jp, jr])).max() < 1e-14


def test_restatement_osc_matches_reference_record():
    """osc_golden.npz replayed: the restatement drives ctrl, the oracle integrates; same gates as the oracle's own replay"""
    from oracle.pyoracle import CtrlCfg
    from robosuite_b200 import controller_config as cc

    g = np.load(os.path.join(ROOT, "tests", "golden", "osc_golden.npz"))
    model = load("Lift_Panda")
    cfg = cc.resolve(model, cc.default_composite_config(), CtrlCfg)
    o = _oracle(model, cfg)
    nsub = int(g["nsub"])
    worst = dict(tau=0.0, goal_pos=0.0, goal_ori=0.0, ctrl=0.0)
    for e in range(g["actions"].shape[0]):
        o.reset_data(); o.qpos[:] = g["qpos0"][e]; o.forward(); o.ctrl_reset()
        st = from_oracle(o.ctrl_state)
        k = 0
        for t in range(g["actions"].shape[1]):
            for sub in range(nsub):
                o.step1()
                r = ref.run(model, cfg, oracle_inputs(o), st, g["actions"][e, t] if sub == 0 else None)
                st = r["state"]
                o.ctrl[:] = r["ctrl"]
                if sub in (0, 1, nsub - 1):
                    gt = g["torques"][e, k]
                    worst["tau"] = max(worst["tau"], np.abs(r["torque"] - gt).max() / np.abs(gt).max())
                    worst["goal_pos"] = max(worst["goal_pos"], np.abs(st["goal_pos"] - g["goal_pos"][e, k]).max())
                    worst["goal_ori"] = max(worst["goal_ori"], np.abs(st["goal_ori"].reshape(3, 3) - g["goal_ori"][e, k]).max())
                    worst["ctrl"] = max(worst["ctrl"], np.abs(r["ctrl"] - g["ctrl"][e, k]).max())
                    k += 1
                o.step2()
    print("restatement vs reference OSC record:", worst)
    assert worst["tau"] < 5e-6 and worst["goal_pos"] < 1e-7 and worst["goal_ori"] < 5e-7 and worst["ctrl"] < 2e-4


def test_restatement_joint_velocity_matches_reference_record():
    """jv_golden.npz replayed substep by substep: clipped torques, goal velocities, ctrl and the anti-windup flag"""
    from oracle.pyoracle import CtrlCfg

    g = np.load(os.path.join(ROOT, "tests", "golden", "jv_golden.npz"))
    model = dedegenerate_sawyer(load("Stack_Sawyer"))
    cfg = ref.make_config(model, "Sawyer", 2, CtrlCfg)
    nsub = int(g["nsub"])
    lo, hi = model.actuator_ctrlrange[:7, 0], model.actuator_ctrlrange[:7, 1]
    worst = 0.0
    for e in range(g["actions"].shape[0]):
        o = _oracle(model, cfg)
        o.qpos[:] = g["qpos0"][e]; o.qvel[:] = 0; o.forward(); o.ctrl_reset()
        st = from_oracle(o.ctrl_state)
        k = 0
        for t in range(g["actions"].shape[1]):
            for sub in range(nsub):
                o.step1()
                r = ref.run(model, cfg, oracle_inputs(o), st, g["actions"][e, t] if sub == 0 else None)
                st = r["state"]
                o.ctrl[:] = r["ctrl"]
                gt = g["torques"][e, k]
                worst = max(worst, np.abs(np.clip(r["torque"], lo, hi) - gt).max() / max(1.0, np.abs(gt).max()))
                assert np.allclose(st["jv"][:7], g["goal_vel"][e, k], rtol=0, atol=1e-12), (e, t, sub)
                assert np.allclose(r["ctrl"], g["ctrl"][e, k], rtol=0, atol=1e-10), (e, t, sub)
                assert bool(st["jv"][66]) == bool(g["saturated"][e, k]), (e, t, sub)
                o.step2()
                k += 1
    print("restatement vs reference JV record: torque rel err %.3g" % worst)
    assert worst < 1e-10


# relative torque gates of the OSC at and near the singular pose: rounding (~1e-16) amplified by the conditioning pinv keeps, 1 / (the
# smallest kept eigenvalue ratio of J M^-1 J^T) ~ 6e6 / 6e10 / 6e14 at near_1e-3 / 1e-5 / 1e-7.  Measured worst against the oracle
# (coupled OSC_POSE, the worst kind): singular 6.3e-11, near_1e-3 2.2e-10, near_1e-5 8.7e-7, near_1e-7 3.9e-3.
NEAR_GATES = {"singular": 1e-9, "near_1e-3": 2e-9, "near_1e-5": 1e-5, "near_1e-7": 5e-2}


def _gate(case, cfg):
    """relative torque gate: rounding, except where pinv's cut-off leaves lambda_full ill-conditioned (module docstring)"""
    return NEAR_GATES.get(case, 1e-12) if cfg.kind in (1, 5) else 1e-12


@pytest.mark.parametrize("conf", CONFIGS, ids=config_id)
def test_restatement_matches_oracle_controller(conf):
    from oracle.pyoracle import CtrlCfg

    robot, kind, over = conf
    model = load(MODELS[robot])
    cfg = ref.make_config(model, robot, kind, CtrlCfg, **over)
    o = _oracle(model, cfg)
    rng = np.random.default_rng(kind + 10 * len(over))
    acts = ref.controlled_actuators(cfg)
    worst = {}
    toggles = 0
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
        st = ref.case_state(model, cfg, case, rng, o.site_xpos, o.site_xmat, o.qpos)
        to_oracle(st, o.ctrl_state)
        action = ref.case_action(cfg, case, rng)
        gate = _gate(case, cfg)
        w = 0.0
        for sub in range(8):
            o.step1()
            inp = oracle_inputs(o)
            o.ctrl_run(action if sub == 0 else None)
            r = ref.run_given_goal(model, cfg, inp, st, action if sub == 0 else None, o.ctrl_state.goal_ori)
            tau = np.array(o.ctrl_state.torques[:cfg.n_arm])
            assert np.isfinite(r["torque"]).all() and np.isfinite(tau).all(), (case, sub)
            err = np.abs(r["torque"] - tau).max() / max(1.0, np.abs(tau).max())
            w = max(w, err)
            assert err < gate, (case, sub, err)
            # ctrl: the clip of the same torques (ill-conditioned torques may land on either side of a limit)
            assert np.allclose(r["ctrl"][acts], o.ctrl[acts], rtol=0, atol=gate * max(1.0, np.abs(tau).max())), (case, sub)
            ost = from_oracle(o.ctrl_state)
            for k in ("goal_pos", "grip"):
                assert np.allclose(r["state"][k], ost[k], rtol=0, atol=1e-12), (case, sub, k)
            assert np.allclose(r["state"]["goal_ori"], ost["goal_ori"], rtol=0, atol=5e-7 if sub == 0 else 0), case  # float32 rounding
            r["state"]["goal_ori"][:] = ost["goal_ori"]
            if kind == 2:
                assert np.allclose(r["state"]["jv"], ost["jv"], rtol=1e-12, atol=1e-12), (case, sub)
                toggles += int(r["state"]["jv"][66] != st["jv"][66])
            elif kind in (3, 4):
                assert np.allclose(r["state"]["jv"][:8], ost["jv"][:8], rtol=0, atol=1e-12), (case, sub)
            st = r["state"]
            o.step2()
        worst[case] = w
    print(config_id(conf), "restatement vs oracle, worst torque rel err per case:", {k: "%.2g" % v for k, v in worst.items()})
    if kind == 2:
        assert toggles > 0  # the anti-windup flag changed within a run
