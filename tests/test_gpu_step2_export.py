"""GPU: the step-2 export (b2s_set_step2_export, BatchedSim.set_step2_export, make(..., dynamics_queries=True)) and the step-2
half of the batched MjData view (every schedule writing the full export's arrays, and the flag changing no other output:
tests/test_gpu_exports.py).

* in the default pipeline configuration, where the late pose load overlays the constraint Jacobian on the last substep, the
  exported arrays agree with themselves: qfrc_constraint = efc_J^T efc_force, qfrc_actuator = gear * actuator_force, and the
  exported qacc passes the solve's optimality certificate on the exported problem (tests/constraint_ref.py, with the gates of
  test_gpu_constraint.py);
* contact_force() is each contact's efc_force rows, and the resting cube's contact forces sum to its weight;
* the errors.

qfrc_constraint = efc_J^T efc_force is held, relative to |efc_J|^T |efc_force|, to 1e-12 in f64 and to QCON_F32 in f32: about 5x
the worst value measured on an H100 80GB HBM3 (700 W power limit) over this file's rollouts (1.1e-7, Stack).  The certificate uses
test_gpu_constraint.py's gates except in f64, where CERT_F64 replaces its 3e-8: that gate was measured on single forward passes, and
in these rollouts PickPlace solves that stopped on the cost improvement ended at up to 4.5e-7 (the solver's stopping tolerance, not
rounding; CERT_F64 is about 5x that).  A row of the exported problem that did not match the solve's would leave a certificate orders of magnitude above
either gate."""
import numpy as np
import pytest

from tests import constraint_ref as cr
from tests.schedules import make_env, random_actions
from tests.test_gpu_constraint import GATES

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

TASKS = ["Lift", "Stack", "Door", "NutAssemblyRound", "PickPlace"]
STEP2 = ("qfrc_actuator", "actuator_force", "qfrc_smooth", "qacc_smooth", "qfrc_constraint", "nefc", "solver_niter",
         "contact_efc_address")
ROWS = ("efc_type", "efc_D", "efc_R", "efc_aref", "efc_force")
QCON_F32 = 5e-7
CERT_F64 = 2e-6


def _blocks(model, efc_type, efc_J, ncon, adr, dim, fric, n, rd):
    """the constraint blocks of one environment's exported rows (tests/constraint_ref.py's structure): the rows before the first
    contact row one block each (friction loss: its dof's bound at the handle's precision), then one block per contact with rows"""
    first = min([int(adr[c]) for c in range(ncon) if adr[c] >= 0] or [n])
    blocks = []
    for r in range(first):
        kind = int(efc_type[r])
        fl = float(rd(model.dof_frictionloss[int(np.argmax(np.abs(efc_J[r])))])) if kind == cr.FRICTION else 0.0
        blocks.append(cr.Block(kind, r, 1, fl=fl))
    for c in range(ncon):
        if adr[c] < 0:
            continue
        d = int(dim[c])
        f3 = fric[c]
        mu = np.array([f3[0], f3[0], f3[1], f3[2], f3[2]])[: d - 1] if d > 1 else None
        blocks.append(cr.Block(cr.ELLIPTIC if d > 1 else cr.FRICTIONLESS, int(adr[c]), d, mu=mu, contact=c))
    return blocks


@pytest.mark.parametrize("precision", ["f32", "f64"])
@pytest.mark.parametrize("task", TASKS)
def test_exported_arrays_agree_under_the_late_pose_overlay(task, precision):
    """default pipeline configuration: the writer runs before the late pose load overlays efc_J"""
    n = 16
    env = make_env(task, n, 1, 7, precision=precision, data_queries=True, dynamics_queries=True)
    sim, m = env.sim, env.model
    acts = random_actions(env, 5, seed=2)
    acts[1:, : n // 2, 2] = -1
    gate = dict(GATES[precision], **({"cert": CERT_F64} if precision == "f64" else {}))
    rd = np.float32 if precision == "f32" else np.float64
    qcon_gate = 1e-12 if precision == "f64" else QCON_F32
    gear = np.asarray(m.actuator_gear)[:, 0]
    dofs = np.asarray(m.jnt_dofadr)[np.asarray(m.actuator_trnid)]
    worst, checked = {"qcon": 0.0, "cert": 0.0, "feas": 0.0}, 0
    for a in acts:
        env.step(a)
        torch.cuda.synchronize()
        h = {k: getattr(sim, k).cpu().numpy() for k in STEP2 + ROWS + ("efc_J", "qM", "qacc", "warn", "ncon", "contact_dim",
                                                                       "contact_friction")}
        # qfrc_actuator: each actuator's force on its own dof, nothing elsewhere (the same product in the handle's precision)
        want = np.zeros_like(h["qfrc_actuator"])
        want[:, dofs] = gear.astype(h["actuator_force"].dtype) * h["actuator_force"]
        assert np.array_equal(h["qfrc_actuator"], want), task
        for e in range(n):
            k = int(h["nefc"][e])
            J, f = h["efc_J"][e, :k].astype(np.float64), h["efc_force"][e, :k].astype(np.float64)
            if k:
                err = np.abs(h["qfrc_constraint"][e] - J.T @ f).max() / max(float((np.abs(J).T @ np.abs(f)).max()), 1e-300)
            else:
                err = float(np.abs(h["qfrc_constraint"][e]).max())
            worst["qcon"] = max(worst["qcon"], err)
            assert err <= qcon_gate, (task, e, err)
            if k == 0 or h["warn"][e] or h["solver_niter"][e] >= m.opt_iterations:
                continue
            ncon = int(h["ncon"][e])
            blocks = _blocks(m, h["efc_type"][e], h["efc_J"][e], ncon, h["contact_efc_address"][e], h["contact_dim"][e],
                             h["contact_friction"][e].astype(np.float64), k, rd)
            assert sum(b.dim for b in blocks) == k, (task, e)
            P = cr.Problem(h["qM"][e], h["qfrc_smooth"][e], J, h["efc_aref"][e, :k], h["efc_R"][e, :k], blocks, m.stat_meaninertia)
            qa = h["qacc"][e].astype(np.float64)
            dist, _ = P.certificate(qa)
            cert = dist / max(1.0, np.sqrt(qa @ P.M @ qa))
            feas = cr.feasibility_violation(blocks, f)
            worst["cert"], worst["feas"] = max(worst["cert"], cert), max(worst["feas"], feas)
            assert cert <= gate["cert"] and feas <= gate["feas"], (task, e, cert, feas)
            checked += 1
    print("%s %s: %d solves, worst %s" % (task, precision, checked, ", ".join("%s %.3g" % kv for kv in sorted(worst.items()))))
    assert checked > 0
    env.close()


def test_contact_force_and_the_resting_cube():
    env = make_env("Lift", 8, 1, 1, precision="f64", dynamics_queries=True)
    sim, m, d = env.sim, env.model, env.sim.data
    zero = torch.zeros((8, env.action_dim), device=env.device, dtype=env.dtype)
    for _ in range(8):
        env.step(zero)
    torch.cuda.synchronize()
    f = d.contact_force().cpu().numpy()
    adr, dim, ncon = (sim.contact_efc_address.cpu().numpy(), sim.contact_dim.cpu().numpy(), sim.ncon.cpu().numpy())
    rows = sim.efc_force.cpu().numpy()
    for e in range(8):
        for c in range(f.shape[1]):
            want = np.zeros(6)
            if c < ncon[e] and adr[e, c] >= 0:
                want[: dim[e, c]] = rows[e, adr[e, c]: adr[e, c] + dim[e, c]]
            assert np.array_equal(f[e, c], want), (e, c)
            assert np.array_equal(d.contact_force(c)[e].cpu().numpy(), want), (e, c)
    frame = sim.contact_frame.cpu().numpy().reshape(8, -1, 3, 3)
    geom = sim.contact_geom.cpu().numpy()
    body = np.asarray(m.geom_bodyid)
    b = env.cube_body_id
    weight = float(np.asarray(m.body_mass)[b]) * -float(np.asarray(m.opt_gravity)[2])
    for e in range(8):
        total = np.zeros(3)
        for c in range(int(ncon[e])):
            g1, g2 = geom[e, c]
            if b in (body[g1], body[g2]):
                world = frame[e, c].T @ f[e, c, :3]  # the force geom1 exerts on geom2
                total += world if body[g2] == b else -world
        assert abs(total[2] - weight) < 1e-3 * weight and np.abs(total[:2]).max() < 1e-3 * weight, (e, total, weight)
    env.close()


def test_errors():
    from robosuite_b200.engine import lib

    env = make_env("Lift", 2, 1, 0)
    env.step(torch.zeros((2, env.action_dim), device=env.device))
    d = env.sim.data
    assert torch.equal(d.qacc, env.sim.qacc)  # state: no export needed
    for call in (lambda: d.qfrc_actuator, lambda: d.efc_force, lambda: d.nefc, lambda: d.contact_force()):
        with pytest.raises(RuntimeError, match="dynamics_queries"):
            call()
    env.sim.set_step2_export(True)
    with pytest.raises(RuntimeError, match="set_contact_export"):
        d.contact_force()
    L = lib()
    assert L.b2s_set_step2_export(None, 1) == -1
    assert b"null handle" in L.b2s_last_error()
    assert L.b2s_set_step2_export(env.sim._h, 1) == 0 and L.b2s_set_step2_export(env.sim._h, 0) == 0
    env.close()
