"""The constraint stage's independent reference (tests/constraint_ref.py) checked on its own, then the CPU oracle checked against it.

The oracle is the yardstick of every other GPU test, and it restates the engine's constraint code line by line like the device does:
an error in how the problem is defined would sit in both.  Here its rows (type, J, aref, R, D, nefc) must equal the reference's,
built from the definitions, to 1e-12; its qacc must pass the reference's optimality certificate; its forces must be f* at its qacc.

The case catalogue (also run on the device by test_gpu_constraint.py) reaches the branches no packaged model reaches: joint limits
with margins (both sides active at once), friction loss in all three Huber zones, every solref / solimp form (negative solref, the
time-constant clamp, power 1 / 2 / 3.5, width 0, dmin == dmax, clamped values), contacts of condim 1, 3, 4 and 6, unequal priority,
solmix 0 / 0.3 / 1 with mixed solref forms, impratio 1 / 20 / 100, the three cone zones, the three Hessian paths (cross-tree,
block-diagonal, same tree) and per-environment geom / dof parameters.
"""
import copy

import numpy as np
import pytest

from tests import constraint_ref as cr
from tests.narrow_phase_ref import axq, compile_scene

ROW_RTOL = 1e-12
# the oracle's answer against the certificate (its solver stops at tolerance 1e-8 on the scaled gradient norm or improvement):
# |qacc - a*|_M <= ORACLE_DIST * max(1, |a*|_M)
ORACLE_DIST = 1e-5


# ------------------------------------------------------------------------------------------------ scenes
def _mjcf(body, impratio=20.0):
    return ('<mujoco><compiler angle="radian" autolimits="true"/><option timestep="0.002" cone="elliptic" impratio="%g"/>'
            '<worldbody>%s</worldbody></mujoco>' % (impratio, body))


# joints: (type, axis, range, margin, extra attributes); one body each, 1 m apart, no contacts
_JOINTS = [
    ("slide", "0 0 1", (-0.1, 0.1), 0.0, 'frictionloss="3"'),
    ("slide", "0 0 1", (-0.1, 0.1), 0.02, 'solimplimit="0.9 0.95 0.01 0.2 1" frictionloss="20" solreffriction="-500 -30"'),
    ("hinge", "0 1 0", (-0.5, 0.5), 0.05, 'solimplimit="0.85 0.99 0.03 0.8 3.5"'),
    ("hinge", "0 1 0", (-0.01, 0.01), 0.03, 'solreflimit="-2000 -50"'),  # narrower than 2 margins: both sides active
    ("slide", "1 0 0", (-0.05, 0.05), 0.01, 'solimplimit="0.9 0.95 0 0.5 2" frictionloss="0.5" solimpfriction="0.5 0.9 0.01 0.3 3"'),
    ("slide", "0 0 1", (-0.05, 0.05), 0.0, 'solimplimit="0.8 0.8 0.01 0.5 2" solreflimit="0.001 1"'),
    ("hinge", "1 0 0", (-0.3, 0.3), 0.01, 'solimplimit="-0.5 1.5 0.02 1.2 0.5"'),
    ("slide", "0 0 1", (-0.2, 0.0), 0.005, 'solimplimit="0.9 0.95 0.05 0.5 2" solreflimit="0.03 0.7" frictionloss="8"'),
]


def joints_scene():
    bodies = []
    for k, (t, ax, rng, margin, extra) in enumerate(_JOINTS):
        bodies.append('<body pos="%d 0 1"><joint type="%s" axis="%s" range="%g %g" margin="%g" %s/>'
                      '<geom type="sphere" size="0.05" pos="0.2 0 0" mass="%g"/></body>' % (k, t, ax, *rng, margin, extra, 0.5 + 0.3 * k))
    return _mjcf("".join(bodies))


def joint_states(model, n, seed):
    """limit violations across the impedance width (below mid, above mid, beyond 1), inactive sides, and velocities that put
    friction loss in each Huber zone"""
    rng = np.random.default_rng(seed)
    Q = np.tile(model.qpos0, (n, 1))
    V = rng.normal(0, 0.6, (n, model.nv))
    for j in range(model.njnt):
        lo, hi = model.jnt_range[j]
        margin = model.jnt_margin[j]
        width = max(float(model.jnt_solimp[j][2]), 0.01)
        mid = min(max(float(model.jnt_solimp[j][3]), 0.05), 0.95)
        for e in range(n):
            x = [0.5 * mid, 0.5 * (1 + mid), 1.5, -0.5][(e + j) % 4]  # violation / width; < 0: inactive
            dist = margin - x * width
            Q[e, model.jnt_qposadr[j]] = lo + dist if (e + 2 * j) % 3 else hi - dist
        if hi - lo < 2 * margin:
            Q[:, model.jnt_qposadr[j]] = rng.uniform(lo - 0.3 * margin, hi + 0.3 * margin, n)
    V[::3] *= 0.02  # slow: friction loss holds (quadratic zone)
    return Q, V


_SIZES = {"box": "0.05 0.04 0.02", "sphere": "0.03", "capsule": "0.02 0.06"}
_HALF = {"box": 0.02, "sphere": 0.03, "capsule": 0.02}


def contact_scene(geom, plane_attr="", geom_attr="", impratio=20.0):
    return _mjcf('<geom type="plane" size="2 2 0.1" %s/><body pos="0 0 0.2"><freejoint/><geom type="%s" size="%s" %s/></body>'
                 % (plane_attr, geom, _SIZES[geom], geom_attr), impratio)


def resting_states(model, n, seed, geoms, spread=0.3):
    """free bodies `geoms` (one per free joint, in order) resting flat on the plane 0.5-3 mm deep, random yaw, velocities that
    separate, slide, spin, roll or press"""
    rng = np.random.default_rng(seed)
    Q = np.tile(model.qpos0, (n, 1))
    V = np.zeros((n, model.nv))
    free = [j for j in range(model.njnt) if model.jnt_type[j] == 0]
    for k, j in enumerate(free):
        a, d = model.jnt_qposadr[j], model.jnt_dofadr[j]
        g = geoms[k]
        for e in range(n):
            Q[e, a + 2] = _HALF[g] - rng.uniform(0.0005, 0.003)
            q = axq([0, 0, 1], rng.uniform(0, 2 * np.pi))
            if g == "capsule":  # lying: one contact per end
                q = _qmul(q, axq([1, 0, 0], np.pi / 2))
            Q[e, a + 3:a + 7] = q
            mode = e % 5
            v = np.zeros(6)
            if mode == 0:
                v[2] = rng.uniform(0.2, 0.5)  # separating: top zone
            elif mode == 1:
                v[:2] = rng.normal(0, spread, 2)  # sliding: middle zone
            elif mode == 2:
                v[2] = -rng.uniform(0.3, 0.8)  # pressing, no slip: bottom zone
            elif mode == 3:
                v[5] = rng.normal(0, 8.0)  # spin about the normal
                v[:2] = rng.normal(0, 0.05, 2)
            else:
                v[3:5] = rng.normal(0, 6.0, 2)  # roll
            V[e, d:d + 6] = v
    return Q, V


def _qmul(a, b):
    w1, x1, y1, z1 = a
    w2, x2, y2, z2 = b
    return np.array([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                     w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2])


# (name, geom, plane attributes, geom attributes, impratio)
CONTACT_VARIANTS = [
    ("sphere_condim1", "sphere", 'condim="1"', 'condim="1"', 20),
    ("box_condim3_impratio1", "box", "", "", 1),
    ("box_condim4", "box", "", 'condim="4" friction="0.8 0.02 0.001"', 20),
    ("capsule_condim6_impratio100", "capsule", "", 'condim="6" friction="0.7 0.03 0.005"', 100),
    ("sphere_plane_condim6", "sphere", 'condim="6" friction="1 0.05 0.01"', "", 20),
    ("box_priority_plane_wins", "box", 'priority="1" friction="0.6 0.01 0.001" solref="0.03 0.9" solimp="0.8 0.9 0.002 0.4 3"',
     'condim="6" friction="1.2 0.1 0.01"', 20),
    ("box_solmix0", "box", 'solmix="0.3" solref="0.01 0.8" solimp="0.85 0.97 0.002 0.3 2"',
     'solmix="0" solref="0.04 1.2" solimp="0.7 0.9 0.005 0.6 4"', 20),
    ("box_solmix03_mixed_solref", "box", 'solref="-8000 -60" solimp="0.9 0.99 0.004 0.5 1"', 'solmix="0.3" solref="0.02 1"', 20),
    ("sphere_negative_solref", "sphere", 'solref="-3000 -40"', 'solref="-5000 -20" condim="4"', 20),
    ("sphere_solmix_both_zero", "sphere", 'solmix="0" solref="0.01 1"', 'solmix="0" solref="0.05 0.5"', 20),
    ("box_timeconst_clamp", "box", 'solref="0.002 1"', 'solref="0.001 1"', 20),
]


def _free(geom, pos, attr=""):
    return '<body pos="%s"><freejoint/><geom type="%s" size="%s" %s/></body>' % (pos, geom, _SIZES[geom], attr)


def stacked_scene():
    return _mjcf('<geom type="plane" size="2 2 0.1"/>' + _free("box", "0 0 0.2") + _free("box", "0 0 0.4", 'condim="4"'))


def stacked_states(model, n, seed):
    """box b on box a on the plane: a contact between two moving trees"""
    Q, V = resting_states(model, n, seed, ["box", "box"])
    rng = np.random.default_rng(seed + 1)
    for e in range(n):
        Q[e, 7:10] = Q[e, 0:3] + [rng.uniform(-0.01, 0.01), rng.uniform(-0.01, 0.01), 0.04 - rng.uniform(0.0005, 0.002)]
        Q[e, 10:14] = Q[e, 3:7]
    return Q, V


def two_on_plane_scene():
    return _mjcf('<geom type="plane" size="2 2 0.1"/>' + _free("sphere", "0 0 0.2", 'condim="4"') + _free("box", "0.5 0 0.2"))


def two_on_plane_states(model, n, seed):
    Q, V = resting_states(model, n, seed, ["sphere", "box"])
    Q[:, 7] += 0.5
    return Q, V


def fingers_scene():
    """a hand on a hinge with two slide-jointed fingers whose pads touch: a contact inside one kinematic tree"""
    return _mjcf('<body pos="0 0 1"><joint type="hinge" axis="0 1 0" damping="1"/><geom type="sphere" size="0.02" contype="0" '
                 'conaffinity="0"/>'
                 '<body pos="-0.03 0 -0.1"><joint type="slide" axis="1 0 0" range="-0.05 0.05" margin="0.004"/>'
                 '<geom type="box" size="0.01 0.02 0.03" condim="4" friction="1 0.02 0.001"/></body>'
                 '<body pos="0.03 0 -0.1"><joint type="slide" axis="1 0 0" range="-0.05 0.05" frictionloss="0.3"/>'
                 '<geom type="box" size="0.01 0.015 0.022" condim="3"/></body></body>')


def fingers_states(model, n, seed):
    rng = np.random.default_rng(seed)
    Q = np.tile(model.qpos0, (n, 1))
    Q[:, 0] = rng.uniform(-0.4, 0.4, n)
    Q[:, 1] = 0.0205 + rng.uniform(0.0, 0.001, n)  # 1-2.5 mm overlap of the two pads (0.04 apart at qpos 0)
    Q[:, 2] = -0.0205 - rng.uniform(0.0, 0.0005, n)
    V = rng.normal(0, 0.3, (n, model.nv))
    return Q, V


_CARRIAGE = '<geom type="sphere" size="0.005" mass="0.2" contype="0" conaffinity="0"/>'
PERENV_BOX = 3  # geom id of the box (after the plane and the two carriages)


def perenv_scene():
    """a box on a chain of slide x (limited, with margin), slide z and hinge y joints: per-environment friction, solref, solimp and
    friction loss (one dof carries both a friction-loss and a limit row)"""
    return _mjcf('<geom type="plane" size="2 2 0.1"/><body pos="0 0 0.02"><joint type="slide" axis="1 0 0" range="-0.01 0.01" '
                 'margin="0.015"/>%s<body><joint type="slide" axis="0 0 1"/>%s<body><joint type="hinge" axis="0 1 0"/>'
                 '<geom type="box" size="0.05 0.04 0.02" condim="4"/></body></body></body>' % (_CARRIAGE, _CARRIAGE))


def perenv_specs(model, n, seed):
    """per environment: {field: {geom: value}} of the box geom and the dof friction loss"""
    rng = np.random.default_rng(seed)
    forms = [[0.02, 1.0], [-4000.0, -50.0], [0.001, 0.7], [0.05, 1.5]]
    imps = [[0.9, 0.95, 0.001, 0.5, 2], [0.5, 0.99, 0.01, 0.2, 1], [0.8, 0.8, 0.01, 0.5, 2], [0.7, 0.95, 0.02, 0.8, 3.5]]
    out = []
    for e in range(n):
        b = PERENV_BOX
        out.append(dict(geom_friction={b: np.array([rng.uniform(0.3, 1.5), rng.uniform(0.001, 0.05), rng.uniform(1e-4, 0.01)])},
                        geom_solref={b: np.array(forms[e % 4])}, geom_solimp={b: np.array(imps[(e // 2) % 4], dtype=np.float64)},
                        dof_frictionloss=np.array([rng.uniform(0, 2), rng.uniform(0, 0.5) * (e % 2), rng.uniform(0, 0.1)])))
    return out


def perenv_states(model, n, seed):
    rng = np.random.default_rng(seed)
    Q = np.zeros((n, model.nq))
    Q[:, 0] = rng.uniform(-0.02, 0.02, n)  # the x limit: inactive, one side, or both sides (range 0.02 < 2 margins)
    Q[:, 1] = -rng.uniform(0.0005, 0.002, n)
    Q[:, 2] = rng.uniform(-0.01, 0.01, n)  # tilted: one or two edge contacts
    V = rng.normal(0, 0.3, (n, model.nv))
    return Q, V


def task_states(name, n, seed, settle=40):
    """a packaged task model and states after oracle settling steps: arm near its home pose, objects dropped onto the table"""
    from oracle.pyoracle import Oracle
    from robosuite_b200.mjcf.compiler import pack_model
    from tests.util import PANDA_INIT, lift_states, load

    model = load(name)
    if name.startswith("Lift"):
        Q, _ = lift_states(model, n, seed)
    else:
        rng = np.random.default_rng(seed)
        Q = np.tile(model.qpos0, (n, 1))
        arm = [j for j, nm in enumerate(model.names["joint"]) if nm and nm.startswith("robot0_") and model.jnt_type[j] == 3]
        for k, j in enumerate(arm):
            Q[:, model.jnt_qposadr[j]] = PANDA_INIT[k] + rng.normal(0, 0.02, n)
        k = 0
        for j in range(model.njnt):
            if model.jnt_type[j] == 0:
                Q[:, model.jnt_qposadr[j] + 1] += 0.12 * k - 0.12
                Q[:, model.jnt_qposadr[j] + 2] += 0.005
                k += 1
    o = Oracle(pack_model(model))
    V = np.zeros((n, model.nv))
    for e in range(n):
        o.reset_data()
        o.qpos[:] = Q[e]
        o.ctrl[:] = 0
        for _ in range(settle):
            o.step()
        Q[e], V[e] = o.qpos, o.qvel
    return model, Q, V


class Case:
    """a scene, per-environment states and (optionally) per-environment parameters"""

    def __init__(self, name, model, Q, V, specs=None):
        self.name, self.model, self.Q, self.V, self.specs = name, model, Q, V, specs
        self.n = len(Q)

    def env(self, e):
        """the per-environment values of environment e as a constraint_ref.Env (without derived constants)"""
        s = self.specs[e] if self.specs else {}
        return cr.Env(dof_frictionloss=s.get("dof_frictionloss"), geom_friction=s.get("geom_friction"), geom_solref=s.get("geom_solref"),
                      geom_solimp=s.get("geom_solimp"))

    def model_of(self, e):
        """the model with environment e's values written in (what the oracle runs)"""
        if not self.specs:
            return self.model
        m = copy.deepcopy(self.model)
        s = self.specs[e]
        for f in ("geom_friction", "geom_solref", "geom_solimp"):
            for g, v in s.get(f, {}).items():
                getattr(m, f)[g] = v
        if s.get("dof_frictionloss") is not None:
            m.dof_frictionloss = np.array(s["dof_frictionloss"], dtype=np.float64)
        return m


def catalogue(n=5, seed=0, packaged=True, n_packaged=2):
    out = []
    m = compile_scene(joints_scene())
    out.append(Case("joints", m, *joint_states(m, max(n, 8), seed)))
    for name, g, pa, ga, imp in CONTACT_VARIANTS:
        m = compile_scene(contact_scene(g, pa, ga, imp))
        out.append(Case(name, m, *resting_states(m, n, seed + len(out), [g])))
    m = compile_scene(stacked_scene())
    out.append(Case("two_boxes_stacked_cross_tree", m, *stacked_states(m, n, seed + 100)))
    m = compile_scene(two_on_plane_scene())
    out.append(Case("two_bodies_on_plane_block_diagonal", m, *two_on_plane_states(m, n, seed + 101)))
    m = compile_scene(fingers_scene())
    out.append(Case("fingers_same_tree", m, *fingers_states(m, n, seed + 102)))
    m = compile_scene(perenv_scene())
    ne = max(n, 8)
    out.append(Case("per_environment_parameters", m, *perenv_states(m, ne, seed + 103), specs=perenv_specs(m, ne, seed + 103)))
    if packaged:
        for task in PACKAGED:
            out.append(Case(task, *task_states(task, n_packaged, seed + 7)))
    return out


_CAT = {}


def cached_catalogue(**kw):
    key = tuple(sorted(kw.items()))
    if key not in _CAT:
        _CAT[key] = catalogue(**kw)
    return _CAT[key]


PACKAGED = ["Lift_Panda", "Stack_Panda", "NutAssemblyRound_Panda"]
CASE_NAMES = (["joints"] + [v[0] for v in CONTACT_VARIANTS] + ["two_boxes_stacked_cross_tree", "two_bodies_on_plane_block_diagonal",
                                                             "fingers_same_tree", "per_environment_parameters"] + PACKAGED)


def case_named(name, **kw):
    return next(c for c in cached_catalogue(**kw) if c.name == name)


# ------------------------------------------------------------------------------------------------ oracle runs
def oracle_forward(model, q, v, warmstart=None):
    from oracle.pyoracle import Oracle
    from robosuite_b200.mjcf.compiler import pack_model

    o = Oracle(pack_model(model))
    o.reset_data()
    o.qpos[:] = q
    o.qvel[:] = v
    o.qacc_warmstart[:] = 0 if warmstart is None else warmstart
    o.forward()
    return o


def rel_err(a, b):
    """largest |a - b| relative to |b| plus the array's own scale"""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    if a.size == 0:
        return 0.0
    return float((np.abs(a - b) / (np.abs(b) + np.abs(b).max() + 1e-300)).max())


def cone_zone(b, f, x, R):
    """'top' (no force), 'bottom' (the unconstrained maximiser is feasible), 'middle' (on the cone's surface)"""
    if not np.any(f):
        return "top"
    return "bottom" if np.allclose(f, -x / R, rtol=1e-9, atol=0) else "middle"


# ------------------------------------------------------------------------------------------------ the reference itself
def test_impedance_at_hand_computed_points():
    si = [0.2, 0.8, 0.1, 0.3, 2.0]
    # x = |pos - margin| / width; below mid: x^2 / mid, above: 1 - (1 - x)^2 / (1 - mid)
    assert cr.impedance(si, -0.01) == pytest.approx(0.2 + 0.6 * 0.01 / 0.3, rel=1e-15)
    assert cr.impedance(si, -0.07) == pytest.approx(0.2 + 0.6 * (1 - 0.09 / 0.7), rel=1e-15)
    assert cr.impedance(si, 0.03, 0.06) == pytest.approx(0.2 + 0.6 * 0.3, rel=1e-15)  # x = mid from either piece
    assert cr.impedance(si, -0.1) == 0.8 and cr.impedance(si, -0.5) == 0.8  # x >= 1
    assert cr.impedance(si, 0.0) == pytest.approx(0.2, abs=1e-300)
    assert cr.impedance([0.2, 0.8, 0.1, 0.3, 3.5], -0.02) == pytest.approx(0.2 + 0.6 * 0.2 ** 3.5 / 0.3 ** 2.5, rel=1e-14)
    assert cr.impedance([0.2, 0.8, 0.1, 0.3, 3.5], -0.09) == pytest.approx(0.2 + 0.6 * (1 - 0.1 ** 3.5 / 0.7 ** 2.5), rel=1e-14)
    assert cr.impedance([0.2, 0.8, 0.1, 0.3, 1.0], -0.06) == pytest.approx(0.2 + 0.6 * 0.6, rel=1e-15)  # power 1: linear
    assert cr.impedance([0.2, 0.8, 0.0, 0.3, 2.0], -0.06) == pytest.approx(0.5, rel=1e-15)  # width 0: flat
    assert cr.impedance([0.7, 0.7, 0.1, 0.3, 2.0], -0.06) == pytest.approx(0.7, rel=1e-15)  # dmin == dmax: flat
    # clamps: dmin, dmax and mid to [1e-4, 0.9999], power to >= 1
    assert cr.impedance([-1, 2, 0.1, 5, 0.2], -0.05) == pytest.approx(1e-4 + (0.9999 - 1e-4) * 0.5, rel=1e-15)
    assert cr.impedance([-1, 2, 0.1, 0.5, 2], -1.0) == 0.9999


def test_stiffness_damping_forms():
    K, B = cr.stiffness_damping([0.02, 1.0], [0.9, 0.95, 0.001, 0.5, 2], 0.002)
    assert K == pytest.approx(1 / (0.95 * 0.02) ** 2, rel=1e-15) and B == pytest.approx(2 / (0.95 * 0.02), rel=1e-15)
    K, B = cr.stiffness_damping([0.001, 0.5], [0.9, 0.95, 0.001, 0.5, 2], 0.002)  # time constant clamped to 2 timesteps
    assert K == pytest.approx(1 / (0.95 * 0.004 * 0.5) ** 2, rel=1e-15) and B == pytest.approx(2 / (0.95 * 0.004), rel=1e-15)
    K, B = cr.stiffness_damping([-3000, -40], [0.9, 0.8, 0.001, 0.5, 2], 0.002)
    assert K == pytest.approx(3000 / 0.64, rel=1e-15) and B == pytest.approx(40 / 0.8, rel=1e-15)


def test_contact_parameter_mixing():
    m = compile_scene(_mjcf('<geom type="plane" size="1 1 0.1" solmix="0.3" condim="4" friction="0.5 0.02 0.003" '
                            'solref="0.01 0.8" solimp="0.8 0.9 0.002 0.3 2"/><body><freejoint/><geom type="sphere" size="0.1" '
                            'solmix="0.7" condim="3" friction="0.9 0.01 0.004" solref="0.03 1.2" solimp="0.6 0.95 0.004 0.5 4"/>'
                            '</body>'))
    dim, f5, sr, si = cr.contact_params(m, 0, 1)
    assert dim == 4 and np.allclose(f5, [0.9, 0.9, 0.02, 0.004, 0.004], rtol=1e-15)
    assert np.allclose(sr, [0.3 * 0.01 + 0.7 * 0.03, 0.3 * 0.8 + 0.7 * 1.2], rtol=1e-14)
    assert np.allclose(si, 0.3 * np.array([0.8, 0.9, 0.002, 0.3, 2]) + 0.7 * np.array([0.6, 0.95, 0.004, 0.5, 4]), rtol=1e-14)
    neg = cr.Env(geom_solref={1: np.array([-100.0, -3.0])})
    assert np.array_equal(cr.contact_params(m, 0, 1, neg)[2], [-100.0, -3.0])  # not both positive: element-wise min
    assert cr.solmix_weight(0, 0) == 0.5 and cr.solmix_weight(0, 1) == 0 and cr.solmix_weight(1, 0) == 1
    m.geom_priority[1] = 2
    dim, f5, sr, si = cr.contact_params(m, 0, 1)
    assert dim == 3 and np.allclose(f5, [0.9, 0.9, 0.01, 0.004, 0.004]) and np.array_equal(sr, [0.03, 1.2])


def test_friction_loss_huber_breakpoints():
    b = cr.Block(cr.FRICTION, 0, 1, fl=2.0)
    R = np.array([0.5])
    for x, f, s in ((-1.0, 2.0, 1.0), (1.0, -2.0, 1.0), (-0.4, 0.8, 0.16), (3.0, -2.0, 5.0)):
        got, cost = cr.forces([b], np.array([x]), R)
        assert got[0] == pytest.approx(f, rel=1e-15) and cost == pytest.approx(s, rel=1e-15)
    # at the breakpoints x = -+R fl, quadratic (x^2 / 2R) and linear (fl |x| - R fl^2 / 2) pieces meet with equal value and slope
    for x in (-1.0, 1.0):
        for h in (1e-7, -1e-7):
            c0 = cr.forces([b], np.array([x]), R)[1]
            c1 = cr.forces([b], np.array([x + h]), R)[1]
            assert (c1 - c0) / h == pytest.approx(-cr.forces([b], np.array([x]), R)[0][0], rel=1e-6)


@pytest.mark.parametrize("dim", [3, 4, 6])
def test_cone_force_against_brute_force(dim):
    """f* of random cone problems: no sampled point of K has a higher objective, and f* is in K"""
    rng = np.random.default_rng(dim)
    for trial in range(40):
        mu = rng.uniform(0.05, 1.5, dim - 1)
        mu[1] = mu[0]
        R0 = rng.uniform(0.01, 2.0)
        R1 = R0 / rng.choice([1.0, 20.0, 100.0])
        R = np.concatenate([[R0], R1 * mu[0] ** 2 / mu ** 2])
        x = rng.normal(0, 1, dim) * rng.uniform(0.1, 3)
        b = cr.Block(cr.ELLIPTIC, 0, dim, mu=mu)
        f, val = cr.forces([b], x, R)
        assert cr.feasibility_violation([b], f) < 1e-14
        assert val == pytest.approx(-(f @ x) - 0.5 * (f * f) @ R, rel=1e-12, abs=1e-15)
        # samples of K: f_0 >= 0, tangential directions scaled onto and inside the cone, plus points around f*
        n = 20000
        f0 = np.abs(rng.normal(0, 1, n)) * np.abs(f[0] + 1) * 2
        d = rng.normal(0, 1, (n, dim - 1))
        d /= np.linalg.norm(d / mu, axis=1, keepdims=True)
        S = np.concatenate([f0[:, None], d * (f0 * rng.uniform(0, 1, n) ** 0.3)[:, None]], axis=1)
        P = f + rng.normal(0, 1e-3, (n, dim)) * (np.abs(f).max() + 1e-3)
        inK = P[:, 0] >= np.linalg.norm(P[:, 1:] / mu, axis=1)
        S = np.concatenate([S, P[inK]])
        vals = -(S @ x) - 0.5 * (S * S) @ R
        assert vals.max() <= val + 1e-12 * max(1.0, abs(val)), (trial, vals.max() - val)


def test_cone_force_equals_zone_formulas():
    """the generic conjugate against the engine's three-zone statement (top: 0; bottom: -x / R; middle: f_0 = -D_0 (x_0 - T)
    / (1 + mu^2) ... with mu = mu_0 sqrt(R_1 / R_0)): equal to rounding, as the substitution h_i = f_i sqrt(R_i) predicts"""
    rng = np.random.default_rng(3)
    seen = set()
    for _ in range(300):
        dim = int(rng.choice([3, 4, 6]))
        mu = rng.uniform(0.1, 1.2, dim - 1)
        mu[1] = mu[0]
        R0 = rng.uniform(0.01, 2.0)
        R1 = R0 / rng.choice([1.0, 20.0])
        R = np.concatenate([[R0], R1 * mu[0] ** 2 / mu ** 2])
        x = rng.normal(0, 1, dim)
        f = cr.cone_force(x, R, mu)
        m = mu[0] * np.sqrt(R1 / R0)
        U = np.concatenate([[x[0] * m], x[1:] * mu])
        N, T = U[0], np.linalg.norm(U[1:])
        if N >= m * T:
            ref, z = np.zeros(dim), "top"
        elif m * N + T <= 0:
            ref, z = -x / R, "bottom"
        else:
            Dm = 1 / R0 / (m * m * (1 + m * m))
            f0 = -Dm * (N - m * T) * m
            ref, z = np.concatenate([[f0], -f0 / T * U[1:] * mu]), "middle"
        seen.add(z)
        assert np.allclose(f, ref, rtol=1e-10, atol=1e-12 * np.abs(ref).max()), (z, f, ref)
    assert seen == {"top", "bottom", "middle"}


def _integrate(model, q, dof, h):
    """qpos moved by h along dof (free joints: position, or the body-frame angular velocity integrated on the quaternion)"""
    q = q.copy()
    for j in range(model.njnt):
        a, d, t = model.jnt_qposadr[j], model.jnt_dofadr[j], model.jnt_type[j]
        if t == 0 and d <= dof < d + 6:
            if dof < d + 3:
                q[a + dof - d] += h
            else:
                w = np.zeros(3)
                w[dof - d - 3] = 1
                q[a + 3:a + 7] = _qmul(q[a + 3:a + 7], axq(w, h))
            return q
        if t in (2, 3) and d == dof:
            q[a] += h
            return q
    raise ValueError(dof)


@pytest.mark.parametrize("scene", ["stacked", "fingers", "Lift_Panda"])
def test_oracle_jacobian_against_finite_differences(scene):
    from oracle.pyoracle import Oracle
    from robosuite_b200.mjcf.compiler import pack_model
    from tests.util import load

    if scene == "stacked":
        m = compile_scene(stacked_scene())
        Q, _ = stacked_states(m, 1, 4)
    elif scene == "fingers":
        m = compile_scene(fingers_scene())
        Q, _ = fingers_states(m, 1, 4)
    else:
        m = load(scene)
        Q = m.qpos0[None] + 0.05
    o = Oracle(pack_model(m))
    q0 = Q[0]
    rng = np.random.default_rng(0)
    h = 1e-6
    for body in range(1, m.nbody):
        o.qpos[:] = q0
        o.kinematics()
        x0, R0 = o.xpos[body].copy(), o.xmat[body].reshape(3, 3).copy()
        pt = x0 + R0 @ rng.normal(0, 0.05, 3)
        jp, jr = o.jac(pt, body)
        local = R0.T @ (pt - x0)
        for dof in range(m.nv):
            P, Rm = [], []
            for s in (1, -1):
                o.qpos[:] = _integrate(m, q0, dof, s * h)
                o.kinematics()
                xb, Rb = o.xpos[body].copy(), o.xmat[body].reshape(3, 3).copy()
                P.append(xb + Rb @ local)
                Rm.append(Rb)
            dp = (P[0] - P[1]) / (2 * h)
            W = (Rm[0] - Rm[1]) / (2 * h) @ R0.T
            dw = np.array([W[2, 1], W[0, 2], W[1, 0]])
            assert np.abs(dp - jp[:, dof]).max() < 1e-7, (scene, body, dof, dp, jp[:, dof])
            assert np.abs(dw - jr[:, dof]).max() < 1e-7, (scene, body, dof, dw, jr[:, dof])


# ------------------------------------------------------------------------------------------------ the oracle against the reference
def reference_of(case, e, o):
    m = case.model_of(e)
    rows = cr.build_rows(m, o)
    return m, rows, cr.problem_from_rows(rows, o.M, o.qfrc_smooth, m.stat_meaninertia)


@pytest.mark.parametrize("name", CASE_NAMES)
def test_oracle_matches_reference(name):
    case = case_named(name)
    worst = dict(rows=0.0, dist=0.0, force=0.0)
    zones = set()
    for e in range(case.n):
        o = oracle_forward(case.model_of(e), case.Q[e], case.V[e])
        m, rows, P = reference_of(case, e, o)
        typ, J, aref, R, D = rows.arrays()
        assert o.nefc == rows.nefc, (e, o.nefc, rows.nefc)
        assert np.array_equal(o.efc("type"), typ), e
        err = max(rel_err(o.efc("J"), J), rel_err(o.efc("aref"), aref), rel_err(o.efc("R"), R), rel_err(o.efc("D"), D))
        worst["rows"] = max(worst["rows"], err)
        assert err < ROW_RTOL, (e, err)
        if rows.nefc == 0:
            continue
        a = np.array(o.qacc)
        astar = P.solve(a)
        dist = np.sqrt((a - astar) @ P.M @ (a - astar)) / max(1.0, np.sqrt(astar @ P.M @ astar))
        worst["dist"] = max(worst["dist"], dist)
        assert dist < ORACLE_DIST, (e, dist)
        x = J @ a - aref
        fstar = P.force(a)
        ferr = rel_err(o.efc("force"), fstar)
        worst["force"] = max(worst["force"], ferr)
        assert ferr < 1e-9, (e, ferr)
        for b in rows.blocks:
            if b.kind == cr.ELLIPTIC:
                zones.add(cone_zone(b, fstar[b.rows], x[b.rows], R[b.rows]))
    print("%s: worst rows %.3g, |qacc - a*|_M %.3g, force %.3g, cone zones %s" % (case.name, worst["rows"], worst["dist"],
                                                                                 worst["force"], sorted(zones)))


def test_catalogue_reaches_every_branch():
    """the catalogue's rows and solutions cover what it is for: both limit sides of one joint at once, every Huber zone of friction
    loss, every cone zone, condim 1 / 3 / 4 / 6, and limits across the impedance width"""
    kinds, zones, huber, dims, both_sides = set(), set(), set(), set(), False
    for case in cached_catalogue(packaged=False):
        for e in range(case.n):
            o = oracle_forward(case.model_of(e), case.Q[e], case.V[e])
            rows = cr.build_rows(case.model_of(e), o)
            typ, J, aref, R, D = rows.arrays()
            x = J @ np.array(o.qacc) - aref
            f = np.array(o.efc("force"))
            lim_dofs = [int(np.flatnonzero(J[b.start])[0]) for b in rows.blocks if b.kind == cr.LIMIT]
            both_sides |= len(lim_dofs) != len(set(lim_dofs))
            for b in rows.blocks:
                kinds.add(b.kind)
                if b.kind == cr.FRICTION:
                    huber.add("linear" if abs(f[b.start]) >= b.fl * (1 - 1e-12) else "quadratic")
                    huber.add("neg" if f[b.start] < 0 else "pos")
                if b.kind in (cr.ELLIPTIC, cr.FRICTIONLESS):
                    dims.add(b.dim)
                if b.kind == cr.ELLIPTIC:
                    zones.add(cone_zone(b, f[b.rows], x[b.rows], R[b.rows]))
    assert kinds == {cr.FRICTION, cr.LIMIT, cr.FRICTIONLESS, cr.ELLIPTIC}
    assert both_sides
    assert huber == {"linear", "quadratic", "neg", "pos"}, huber
    assert zones == {"top", "middle", "bottom"}, zones
    assert dims == {1, 3, 4, 6}, dims
