"""The device's smooth dynamics (kinematics, velocity stage, composite inertia, actuation, the M solves and the Euler step) against the
independent fp64 reference of tests/dynamics_ref.py, on the case catalogue of test_cpu_dynamics.py: one environment per state, one
`BatchedSim.forward()` with export.

- forward(), f64 and f32, every case: body, site and colliding-geom poses (xquat up to sign), cdof, qM, qfrc_bias, qfrc_passive,
  qfrc_actuator, actuator_force, qfrc_smooth and qacc_smooth (by its residual M a - qfrc_smooth, see compare_forward).
- One step(1) of the contact-free scenes from the same state against the reference's Euler step (the velocity update by its
  residual, the position update against the reference's integration of the device's velocity), and 200 f64 substeps against the
  reference's trajectory.
- Modes 0 (fused), 1 (phase pipeline) and 2 (unit queue) give bit-identical qpos / qvel on every contact-free scene.
- The Door's latch spring on the device, and the model checks of b2s_create (host side).

Errors are relative (rel_err of test_cpu_dynamics.py).  f64 is held to 1e-12 throughout.  The f32 gates are about 5x the worst
values measured on an H100 80GB HBM3 (700 W power limit) over this file's cases (worst case in brackets):
    poses 6.9e-7 (tree_32 site_xmat), cdof 5.0e-7 (tree_32), qM 1.1e-6 (PickPlace_Panda), qfrc_bias 3.0e-6 (gravity_zero),
    qfrc_passive 2.0e-6 (fluid_wind), qfrc_actuator 3.3e-8 (actuators), actuator_force 1.7e-8 (Lift_Panda), qfrc_smooth 3.0e-6
    (gravity_zero), qacc_smooth residual 5.5e-6 (fluid_wind), one step 1.2e-4 (gravity_zero's velocity residual: with no gravity its
    force is only the gyroscopic term, so the relative error is large).
The f64 forward outputs measured at most 1.4e-14 and one f64 step at most 1.9e-13; the 200-substep f64 trajectories at most 1.3e-13
(fluid_wind), gated at 1e-12.
"""
import numpy as np
import pytest

from tests import dynamics_ref as dr
from tests.schedules import switches
from tests.test_cpu_dynamics import CASE_NAMES, GPU_CAPACITY, SCENES, case_named, compare_forward, rel_err, step_errors

pytestmark = pytest.mark.gpu

F64 = 1e-12
GATES_F32 = dict(pose=3.5e-6, cdof=2.5e-6, M=5.5e-6, qfrc_bias=1.5e-5, qfrc_passive=1e-5, qfrc_actuator=1.7e-7, actuator_force=1e-7,
                 qfrc_smooth=1.5e-5, qacc_smooth=2.8e-5, step=6e-4)
TRAJ_F64 = 1e-12
N_ENV = 4
# the packaged tasks at the catalogue's states hold more contacts than the default capacities (32 contacts, 64 rows)
CAPACITY = {"NutAssemblyRound_Panda": (128, 384), "Stack_Panda": (64, 256), "Lift_Panda": (64, 256), "PickPlace_Panda": (128, 384),
            "Door_Panda": (64, 256), "Lift_Sawyer": (64, 256)}
_POSE = {"xpos", "xmat", "site_xpos", "site_xmat", "geom_xpos", "geom_xmat", "xquat"}


def _case(name):
    return case_named(name, n=N_ENV)


def _gate(prec, field):
    if prec == "f64":
        return F64
    return GATES_F32["pose" if field in _POSE else "M" if field == "M" else field]


def make_sim(case, prec):
    import torch

    from robosuite_b200.engine import BatchedSim

    mc, me = CAPACITY.get(case.name, GPU_CAPACITY)
    sim = BatchedSim(case.model, case.n, precision=prec, maxcon=mc, maxefc=me)
    t = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float64), dtype=sim.dtype)
    if case.envs:
        for b in case.envs[0]["body_mass"]:
            sim.model_override("body_mass", b).copy_(t([v["body_mass"][b] for v in case.envs]))
            sim.model_override("body_inertia", b).copy_(t([v["body_inertia"][b] for v in case.envs]))
        sim.model_override("dof_damping").copy_(t([v["dof_damping"] for v in case.envs]))
        sim.model_override("dof_armature").copy_(t([v["dof_armature"] for v in case.envs]))
        sim.set_const()
    sim.qpos.copy_(t(case.Q))
    sim.qvel.copy_(t(case.V))
    if case.model.nu:
        sim.ctrl.copy_(t(case.U))
    return sim, t


def device_forward(case, prec):
    import torch

    sim, _ = make_sim(case, prec)
    try:
        sim.forward()
        torch.cuda.synchronize()
        get = lambda k: sim.array(k).cpu().numpy().astype(np.float64)
        out = {k: get(k) for k in ("xpos", "xquat", "xmat", "site_xpos", "site_xmat", "geom_xpos", "geom_xmat", "cdof", "qM", "qfrc_bias",
                                   "qfrc_passive", "qfrc_actuator", "actuator_force", "qfrc_smooth", "qacc_smooth")}
        out["warn"] = sim.array("warn").cpu().numpy().astype(np.int64)
        return out
    finally:
        sim.close()


def _colliding_geoms(m):
    return sorted(set(np.asarray(m.pair_geom).reshape(-1).tolist()))


@pytest.mark.parametrize("prec", ["f64", "f32"])
@pytest.mark.parametrize("name", CASE_NAMES)
def test_forward_matches_reference(name, prec):
    case = _case(name)
    dev = device_forward(case, prec)
    # contact capacity warnings (bits 4, 8) of the packaged models at these states do not touch the smooth dynamics
    assert int(np.abs(dev["warn"] & ~(12 if case.contacts else 0)).max()) == 0, dev["warn"]
    names = {"M": "qM"}
    worst, bad = {}, []
    cg = _colliding_geoms(case.model)
    for e in range(case.n):
        f = case.forward(e)
        errs = compare_forward(f, lambda k: dev[names.get(k, k)][e], dev["xquat"][e])
        if cg:
            errs["geom_xpos"] = rel_err(dev["geom_xpos"][e][cg], f.geom_xpos[cg])
            errs["geom_xmat"] = rel_err(dev["geom_xmat"][e][cg].reshape(-1, 3, 3), f.geom_xmat[cg])
        for k, v in errs.items():
            worst[k] = max(worst.get(k, 0.0), v)
            if not v <= _gate(prec, k):
                bad.append((e, k, v))
    print("%s %s: %s" % (name, prec, ", ".join("%s %.3g" % kv for kv in sorted(worst.items()))))
    assert not bad, bad[:8]


@pytest.mark.parametrize("prec", ["f64", "f32"])
@pytest.mark.parametrize("name", SCENES)
def test_one_step_matches_reference_euler(name, prec):
    import torch

    case = _case(name)
    sim, _ = make_sim(case, prec)
    try:
        sim.step(1)
        torch.cuda.synchronize()
        assert int(sim.warn.abs().max()) == 0
        q1, v1 = sim.qpos.cpu().numpy().astype(np.float64), sim.qvel.cpu().numpy().astype(np.float64)
    finally:
        sim.close()
    gate = F64 if prec == "f64" else GATES_F32["step"]
    worst = {}
    for e in range(case.n):
        errs = step_errors(case.forward(e), q1[e], v1[e])
        for k, v in errs.items():
            worst[k] = max(worst.get(k, 0.0), v)
    print("%s %s step: %s" % (name, prec, ", ".join("%s %.3g" % kv for kv in sorted(worst.items()))))
    assert max(worst.values()) <= gate, worst


# free_bodies is left out: explicit Euler on its fast anisotropic spins gains energy, which amplifies rounding over 200 substeps
_TRAJ = ["hinge_chain", "slide_hinge_mix", "fluid_wind", "springs", "actuators", "gravity_tilted", "tree_9"]


@pytest.mark.parametrize("name", _TRAJ)
def test_f64_trajectory_matches_reference(name):
    """200 substeps (0.4 s) from the catalogue's first state, ctrl held"""
    import torch

    case = _case(name)
    sim, _ = make_sim(case, "f64")
    n = 200
    try:
        sim.step(n)
        torch.cuda.synchronize()
        assert int(sim.warn.abs().max()) == 0
        qd, vd = sim.qpos.cpu().numpy()[0], sim.qvel.cpu().numpy()[0]
    finally:
        sim.close()
    q, v = case.Q[0].copy(), case.V[0].copy()
    for _ in range(n):
        q, v = dr.Forward(case.model, q, v, case.U[0]).euler()
    err = max(float(np.abs(qd - q).max() / max(1.0, np.abs(q).max())), float(np.abs(vd - v).max() / max(1.0, np.abs(v).max())))
    print("%s trajectory f64: %.3g" % (name, err))
    assert err <= TRAJ_F64, err


@pytest.mark.parametrize("prec", ["f64", "f32"])
@pytest.mark.parametrize("name", SCENES)
def test_schedules_bit_exact_on_dynamics_scenes(name, prec):
    import torch

    case = _case(name)
    res = []
    for mode in (0, 1, 2):
        with switches(gjk_cache=False):
            sim, _ = make_sim(case, prec)
            try:
                sim.set_mode(mode)
                sim.step(20)
                torch.cuda.synchronize()
                assert int(sim.warn.abs().max()) == 0
                res.append((sim.qpos.cpu().numpy().copy(), sim.qvel.cpu().numpy().copy()))
            finally:
                sim.close()
    assert np.abs(res[0][0] - case.Q).max() > 0
    for mode in (1, 2):
        assert np.array_equal(res[0][0], res[mode][0]) and np.array_equal(res[0][1], res[mode][1]), mode


@pytest.mark.parametrize("prec", ["f64", "f32"])
def test_door_latch_spring(prec):
    """the latch (stiffness 1, springref 0) pulls back in proportion to its angle: the device's passive force on its dof equals the
    reference's, which holds -stiffness q beside damping and fluid terms"""
    case = _case("Door_Panda")
    m = case.model
    j = m.name2id("joint", "Door_latch_joint")
    d, a = int(m.jnt_dofadr[j]), int(m.jnt_qposadr[j])
    assert m.jnt_stiffness[j] == 1 and np.all(np.abs(case.Q[:, a]) > 0.3)
    dev = device_forward(case, prec)
    tol = 1e-12 if prec == "f64" else 1e-5
    for e in range(case.n):
        f = case.forward(e)
        spring = -m.jnt_stiffness[j] * (case.Q[e, a] - m.qpos_spring[a])
        assert abs(f.qfrc_spring_damper[d] - (spring - m.dof_damping[d] * case.V[e, d])) <= 1e-15
        assert abs(dev["qfrc_passive"][e, d] - f.qfrc_passive[d]) <= tol * max(1.0, abs(f.qfrc_passive[d])), (e, dev["qfrc_passive"][e, d],
                                                                                                             f.qfrc_passive[d])


def _reject_models():
    from tests.narrow_phase_ref import compile_scene
    from tests.test_cpu_dynamics import _mjcf

    body = '<inertial pos="0 0 0" mass="1" diaginertia="0.1 0.1 0.1"/>'
    ball = compile_scene(_mjcf('<body><joint type="ball"/>%s</body>' % body))
    two = compile_scene(_mjcf('<body><joint type="hinge"/><joint type="slide"/>%s</body>' % body))
    inner = ""
    for _ in range(65):
        inner = '<body pos="0 0 -0.1"><joint type="hinge" axis="0 1 0"/>%s%s</body>' % (body, inner)
    big = compile_scene(_mjcf(inner))
    free = compile_scene(_mjcf('<body><freejoint/>%s</body>' % body))
    free.jnt_stiffness = np.array([2.0])  # the compiler refuses this; the library checks models it did not compile too
    return [("ball", ball, "ball joints"), ("two joints", two, "more than one joint"), ("nv 65", big, "nv > 64"),
            ("free stiffness", free, "stiffness on a free joint")]


def test_create_rejects_unsupported_models():
    from robosuite_b200.engine import B2SError, BatchedSim

    for label, m, msg in _reject_models():
        with pytest.raises(B2SError, match=msg):
            BatchedSim(m, 2, precision="f64")
    ok = case_named("springs", n=N_ENV).model
    sim = BatchedSim(ok, 2, precision="f64")
    sim.close()
