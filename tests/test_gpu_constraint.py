"""The device's constraint stage (row assembly `make_constraint` and the primal Newton `solve`) against the independent fp64
reference of tests/constraint_ref.py, on the case catalogue of test_cpu_constraint.py: one environment per state, one
`BatchedSim.forward()` with export, `qacc_warmstart` set before it.

- Rows: nefc, efc_type, efc_J, efc_aref, efc_R and efc_D against the reference's rows, built from the oracle's fp64 state (contact
  frames and positions are the oracle's; the narrow-phase tests pin the device's against them).
- Solve, on the device's own exported problem (qM, qfrc_smooth, efc_*, contact_friction cast to fp64): the optimality certificate
  |g(qacc)|_{M^-1} at the exported qacc, efc_force = f*(qacc), qfrc_constraint = J^T efc_force, and feasible forces.  This
  judges the solver apart from assembly rounding.
- End to end: qacc against the reference minimiser a*, efc_force against f*(a*).
- Warm start at 0, qacc_smooth, a* and a far-off vector: the same answer within the gates; f64 from a* ends within one iteration.
- Capacity: with a row budget one contact does not fit, warn bit 8 is set, the kept contacts are exactly a prefix, and the solve
  matches the reference over the kept rows.
- Schedules: modes 0, 1 and 2 give bit-identical qpos / qvel after `step(n)` on the new scenes, with and without a small tail tier
  (4 contacts, 8 rows beyond friction loss) that sends the larger environments to the large tier.

Errors are relative: rows and forces to |ref| plus the array's own scale; qacc - a* and the certificate in the M-norm, to max(1, |a|_M).
Gates per precision and quantity (GATES).  f64 rows are held to 1e-12; the other gates are about 5x the worst values measured on an
H100 80GB HBM3 (700 W power limit) over this file's cases (qcon and feasibility in f64: 1e-14, above rounding):
          rows     certificate  qacc e2e  force e2e  force = f*(qacc)  qfrc_constraint  feasibility
    f64   1.3e-14  5.6e-9       1.3e-9    2.8e-9     4.3e-13           9.3e-17          2.4e-16
    f32   8.2e-5   4.7e-4       2.7e-4    5.9e-5     1.5e-4            2.6e-7           9.6e-8
The f64 certificate and end-to-end errors sit at the solver's stopping tolerance (1e-8 on the scaled gradient norm or cost
improvement), not at rounding.  The f32 worsts come from stiff contacts: the stacked boxes and the resting box (certificate,
forces), the two finger pads inside one tree (qacc), and the joint limits' rows (aref and R from fp32 positions).  No case family needs a looser gate.
"""
import numpy as np
import pytest

from tests import constraint_ref as cr
from tests.test_cpu_constraint import CASE_NAMES, case_named, oracle_forward, rel_err

pytestmark = pytest.mark.gpu

GATES = {
    "f64": dict(rows=1e-12, cert=3e-8, qacc=6e-9, force=1.5e-8, fstar=2e-12, qcon=1e-14, feas=1e-14),
    "f32": dict(rows=4e-4, cert=2.5e-3, qacc=1.5e-3, force=3e-4, fstar=8e-4, qcon=1.5e-6, feas=5e-7),
}
N_ENV = 8
# the packaged tasks' settled states hold more contacts than the default capacities (32 contacts, 64 rows)
CAPACITY = {"NutAssemblyRound_Panda": (128, 384), "Stack_Panda": (64, 256), "Lift_Panda": (64, 256)}


def _case(name):
    return case_named(name, n=N_ENV, seed=11, packaged=True, n_packaged=4)


# ------------------------------------------------------------------------------------------------ device runs
def device_forward(case, prec, warm=None, maxefc=None):
    """one forward() of one environment per state; returns a dict of host fp64 arrays (and the derived constants per env)"""
    import torch

    from robosuite_b200.engine import BatchedSim

    maxcon, me = CAPACITY.get(case.name, (None, None))
    sim = BatchedSim(case.model, case.n, precision=prec, maxcon=maxcon, maxefc=maxefc or me)
    try:
        dt = sim.dtype
        t = lambda a: torch.as_tensor(np.asarray(a), dtype=dt)
        if case.specs:
            for f in ("geom_friction", "geom_solref", "geom_solimp"):
                for g in case.specs[0][f]:
                    sim.model_override(f, g).copy_(t([s[f][g] for s in case.specs]))
            sim.model_override("dof_frictionloss").copy_(t([s["dof_frictionloss"] for s in case.specs]))
            sim.set_const()
        sim.qpos.copy_(t(case.Q))
        sim.qvel.copy_(t(case.V))
        sim.qacc_warmstart.copy_(t(np.zeros((case.n, case.model.nv)) if warm is None else warm))
        sim.forward()
        torch.cuda.synchronize()
        get = lambda name: sim.array(name).cpu().numpy().astype(np.float64)
        out = {k: get(k) for k in ("qacc", "qM", "qfrc_smooth", "qacc_smooth", "qfrc_constraint", "efc_J", "efc_aref", "efc_R",
                                   "efc_D", "efc_force", "contact_friction", "contact_dist")}
        for k in ("nefc", "efc_type", "warn", "solver_niter", "ncon"):
            out[k] = sim.array(k).cpu().numpy().astype(np.int64)
        if case.specs:
            for k in ("dof_invweight0", "body_invweight0", "meaninertia"):
                out[k] = get(k)
        return out
    finally:
        sim.close()


class Ref:
    """the reference of one environment: oracle state, rows, problem and minimiser"""

    def __init__(self, case, e, dev=None, max_rows=None):
        self.model = case.model_of(e)
        self.o = oracle_forward(self.model, case.Q[e], case.V[e])
        env = case.env(e)
        mi = self.model.stat_meaninertia
        if dev is not None and "dof_invweight0" in dev:  # overrides declared: the environment's own derived constants
            env.dof_invweight0, env.body_invweight0 = dev["dof_invweight0"][e], dev["body_invweight0"][e]
            mi = float(dev["meaninertia"][e])
        self.meaninertia = mi
        self.rows = cr.build_rows(self.model, self.o, env, max_rows=max_rows)
        self.P = cr.problem_from_rows(self.rows, self.o.M, self.o.qfrc_smooth, mi)
        self._astar = None

    @property
    def astar(self):
        if self._astar is None:
            self._astar = self.P.solve(np.array(self.o.qacc))
        return self._astar


_REFS = {}


def refs_of(case, dev, max_rows=None):
    key = (case.name, max_rows)
    if key not in _REFS:
        _REFS[key] = [Ref(case, e, dev, max_rows) for e in range(case.n)]
    return _REFS[key]


def device_problem(ref, dev, e, prec):
    """the device's exported problem of environment e in fp64, with the reference's block structure (friction-loss bounds at the
    device's precision, cone coefficients from the device's contact_friction)"""
    n = int(dev["nefc"][e])
    rd = np.float32 if prec == "f32" else np.float64
    blocks = []
    for b in ref.rows.blocks:
        mu = None
        if b.kind == cr.ELLIPTIC:
            f3 = dev["contact_friction"][e, b.contact]
            mu = np.array([f3[0], f3[0], f3[1], f3[2], f3[2]])[:b.dim - 1]
        blocks.append(cr.Block(b.kind, b.start, b.dim, fl=float(rd(b.fl)), mu=mu, contact=b.contact))
    return cr.Problem(dev["qM"][e], dev["qfrc_smooth"][e], dev["efc_J"][e, :n], dev["efc_aref"][e, :n], dev["efc_R"][e, :n], blocks,
                      ref.meaninertia)


def m_dist(P, a, b):
    d = a - b
    return float(np.sqrt(max(d @ P.M @ d, 0.0)) / max(1.0, np.sqrt(max(b @ P.M @ b, 0.0))))


def check_env(ref, dev, e, prec, worst, bad, tag, rows=True, e2e=True):
    g = GATES[prec]
    n = int(dev["nefc"][e])
    typ, J, aref, R, D = ref.rows.arrays()

    def gate(name, val):
        worst[name] = max(worst.get(name, 0.0), val)
        if not val <= g[name]:
            bad.append((tag, e, name, val))

    if n != ref.rows.nefc or not np.array_equal(dev["efc_type"][e, :n], typ):
        bad.append((tag, e, "rows", "nefc %d vs %d, types %s vs %s" % (n, ref.rows.nefc, dev["efc_type"][e, :n].tolist(), typ.tolist())))
        return
    if rows:
        gate("rows", max(rel_err(dev["efc_J"][e, :n], J), rel_err(dev["efc_aref"][e, :n], aref), rel_err(dev["efc_R"][e, :n], R),
                         rel_err(dev["efc_D"][e, :n], D)))
    if n == 0:
        return
    P = device_problem(ref, dev, e, prec)
    a, f = dev["qacc"][e], dev["efc_force"][e, :n]
    dist, _ = P.certificate(a)
    gate("cert", dist / max(1.0, np.sqrt(a @ P.M @ a)))
    gate("fstar", rel_err(f, P.force(a)))
    gate("qcon", rel_err(dev["qfrc_constraint"][e], P.J.T @ f))
    gate("feas", cr.feasibility_violation(P.blocks, f))
    if e2e:
        astar = ref.astar
        gate("qacc", m_dist(ref.P, a, astar))
        gate("force", rel_err(f, ref.P.force(astar)))


def report(tag, prec, worst):
    print("%s %s: " % (tag, prec) + ", ".join("%s %.3g" % kv for kv in sorted(worst.items())))


@pytest.mark.parametrize("prec", ["f64", "f32"])
@pytest.mark.parametrize("name", CASE_NAMES)
def test_constraint_stage_matches_reference(name, prec):
    case = _case(name)
    dev = device_forward(case, prec)
    assert int(np.abs(dev["warn"]).max()) == 0, dev["warn"]
    refs = refs_of(case, dev)
    worst, bad = {}, []
    for e in range(case.n):
        check_env(refs[e], dev, e, prec, worst, bad, case.name)
    report(case.name, prec, worst)
    assert not bad, bad[:8]


def test_joint_limit_margin_both_sides_active():
    """a hinge whose range is narrower than twice its margin: both limit rows in one environment, with pos - margin in impedance
    and aref, against the reference and the oracle (before the device honoured jnt_margin it built no row here)"""
    from tests.narrow_phase_ref import compile_scene
    from tests.test_cpu_constraint import Case, _mjcf

    m = compile_scene(_mjcf('<body pos="0 0 1"><joint type="hinge" axis="0 1 0" range="-0.01 0.02" margin="0.03" '
                            'solimplimit="0.8 0.95 0.05 0.4 3" solreflimit="0.02 0.8"/><geom type="sphere" size="0.05" pos="0.2 0 0"/>'
                            '</body>'))
    case = Case("margin", m, np.array([[0.005], [-0.005], [0.012]]), np.array([[0.3], [-0.2], [0.0]]))
    for prec in ("f64", "f32"):
        dev = device_forward(case, prec)
        assert int(np.abs(dev["warn"]).max()) == 0
        refs = [Ref(case, e) for e in range(case.n)]
        for e, r in enumerate(refs):
            assert r.o.nefc == 2 and r.rows.nefc == 2 and list(dev["nefc"][e:e + 1]) == [2], (prec, e, dev["nefc"])
            assert np.array_equal(dev["efc_J"][e, :2, 0], [1.0, -1.0])
            tol = GATES[prec]["rows"]
            for k, ok in (("aref", "aref"), ("R", "R"), ("D", "D")):
                assert rel_err(dev["efc_" + k][e, :2], r.o.efc(ok)) < tol, (prec, e, k, dev["efc_" + k][e, :2], r.o.efc(ok))
            worst, bad = {}, []
            check_env(r, dev, e, prec, worst, bad, "margin")
            assert not bad, bad


_WARM_CASES = ["joints", "box_condim4", "two_boxes_stacked_cross_tree", "fingers_same_tree", "per_environment_parameters", "Lift_Panda"]


@pytest.mark.parametrize("prec", ["f64", "f32"])
@pytest.mark.parametrize("name", _WARM_CASES)
def test_warm_start_gives_the_same_answer(name, prec):
    case = _case(name)
    dev0 = device_forward(case, prec)
    refs = refs_of(case, dev0)
    astar = np.array([r.astar for r in refs])
    rng = np.random.default_rng(2)
    starts = {"zero": None, "qacc_smooth": dev0["qacc_smooth"], "astar": astar,
              "far": astar + rng.normal(0, 100.0, astar.shape) * (1 + np.abs(astar))}
    worst, bad = {}, []
    for label, w in starts.items():
        dev = device_forward(case, prec, warm=w)
        assert int(np.abs(dev["warn"]).max()) == 0, (label, dev["warn"])
        for e in range(case.n):
            check_env(refs[e], dev, e, prec, worst, bad, label, rows=False)
        if label == "astar" and prec == "f64":
            assert int(dev["solver_niter"].max()) <= 1, dev["solver_niter"]
    report(name + " warm starts", prec, worst)
    assert not bad, bad[:8]


@pytest.mark.parametrize("prec", ["f64", "f32"])
def test_capacity_keeps_a_prefix_of_contacts(prec):
    """box_condim4 rests on four corner contacts of four rows each; a budget of ten rows keeps the first two contacts"""
    case = _case("box_condim4")
    budget = 10
    dev = device_forward(case, prec, maxefc=budget)
    refs = refs_of(case, dev, max_rows=budget)
    worst, bad = {}, []
    dropped = 0
    for e in range(case.n):
        full = len([c for c in refs[e].o.contacts() if c["dist"] < 0])
        kept = len(refs[e].rows.blocks)
        if full * 4 > budget:
            dropped += 1
            assert int(dev["warn"][e]) & 8, (e, dev["warn"][e])
        assert int(dev["nefc"][e]) == 4 * kept, (e, dev["nefc"][e], kept)
        check_env(refs[e], dev, e, prec, worst, bad, "capacity")
    report("capacity", prec, worst)
    assert dropped > 0
    assert not bad, bad[:8]


_SCHEDULE_CASES = ["joints", "sphere_condim1", "capsule_condim6_impratio100", "two_boxes_stacked_cross_tree", "fingers_same_tree",
                   "per_environment_parameters"]


def _steps(case, mode, prec, tier_small, n=20):
    import os

    import torch

    from robosuite_b200.engine import BatchedSim

    os.environ["B2S_NO_GJK_CACHE"] = "1"  # the fused kernel has no GJK warm start
    maxcon, me = CAPACITY.get(case.name, (None, None))
    sim = BatchedSim(case.model, case.n, precision=prec, maxcon=maxcon, maxefc=me, tier_small=tier_small)
    try:
        dt = sim.dtype
        t = lambda a: torch.as_tensor(np.asarray(a), dtype=dt)
        if case.specs:
            for f in ("geom_friction", "geom_solref", "geom_solimp"):
                for g in case.specs[0][f]:
                    sim.model_override(f, g).copy_(t([s[f][g] for s in case.specs]))
            sim.model_override("dof_frictionloss").copy_(t([s["dof_frictionloss"] for s in case.specs]))
            sim.set_const()
        sim.set_mode(mode)
        sim.qpos.copy_(t(case.Q))
        sim.qvel.copy_(t(case.V))
        sim.step(n)
        torch.cuda.synchronize()
        assert int(sim.warn.abs().max()) == 0
        return sim.qpos.cpu().numpy().copy(), sim.qvel.cpu().numpy().copy()
    finally:
        sim.close()
        os.environ.pop("B2S_NO_GJK_CACHE", None)


@pytest.mark.parametrize("prec", ["f64", "f32"])
@pytest.mark.parametrize("name", _SCHEDULE_CASES)
def test_schedules_bit_exact_on_constraint_scenes(name, prec):
    """modes 0 (fused), 1 (phase pipeline) and 2 (unit queue), each with and without a small tail tier (4 contacts, 8 rows beyond
    friction loss) that sends the larger environments to the large tier: bit-identical qpos and qvel"""
    case = _case(name)
    a = _steps(case, 0, prec, None)
    assert np.isfinite(a[0]).all() and np.abs(a[0] - case.Q).max() > 0
    for mode in (1, 2):
        for tier in (None, (4, 8)):
            b = _steps(case, mode, prec, tier)
            assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]), (mode, tier)
