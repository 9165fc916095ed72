"""The smooth dynamics' independent reference (tests/dynamics_ref.py) checked on its own, then the CPU oracle checked against it.

The oracle is the yardstick of the GPU tests, and it restates the device's formulation (world-origin spatial algebra, 10-number
inertias, the same hinge-about-anchor composition, the same fluid code): a definition error would sit in both.  Here the reference
first passes checks that need no engine at all (finite-differenced kinematics, the mass matrix as a sum of body Jacobians, kinetic
energy, the Lagrangian bias, closed forms of a lone body, the fluid model at hand-set velocities, two known Euler answers), then the
oracle must equal it to 1e-12 on every case of the catalogue below (also run on the device by test_gpu_dynamics.py).

The catalogue has the contact pairs disabled, so only the smooth dynamics runs, and reaches what no packaged model does: slide joints
inside chains, ref != 0, a hinge below a free body, off-diagonal full inertias (non-identity iquat), joint anchors away from the body
origin, a massive dof-less body welded inside a chain, joint springs with springref != ref, fluid forces with wind, velocity and
general-affine actuators with gear != 1 and the ctrl / force clamps, tilted and zero gravity, every branch of the device's M solve
(block-diagonal solves for trees of 8, 9 and 12 dofs, register solves for 16, 24 and 32, the dense Cholesky for nv 33 to 64), more
than 64 bodies and a tree deeper than 32 levels, and per-environment masses, inertias, damping and armature.
"""
import numpy as np
import pytest

from tests import dynamics_ref as dr
from tests.narrow_phase_ref import compile_scene

ORACLE_RTOL = 1e-12
_OFF = 'contype="0" conaffinity="0"'


# ------------------------------------------------------------------------------------------------ scenes
def _mjcf(body, option="", actuator=""):
    return ('<mujoco><compiler angle="radian" autolimits="true"/><option timestep="0.002" cone="elliptic" %s/><worldbody>%s</worldbody>'
            '<actuator>%s</actuator></mujoco>' % (option, body, actuator))


def _v(x):
    return " ".join("%.6g" % float(t) for t in np.ravel(x))


def _inertial(rng, full=False, mass=None):
    mass = rng.uniform(0.3, 2.0) if mass is None else mass
    if full:
        A = rng.normal(0, 1, (3, 3))
        I = A @ A.T * 0.01 + np.eye(3) * 0.01
        return '<inertial pos="%s" mass="%.6g" fullinertia="%s"/>' % (_v(rng.uniform(-0.05, 0.05, 3)), mass,
                                                                       _v([I[0, 0], I[1, 1], I[2, 2], I[0, 1], I[0, 2], I[1, 2]]))
    d = rng.uniform(0.005, 0.03, 3)
    return '<inertial pos="%s" mass="%.6g" diaginertia="%s"/>' % (_v(rng.uniform(-0.05, 0.05, 3)), mass, _v(d))


def _quat(rng):
    q = rng.normal(0, 1, 4)
    return q / np.linalg.norm(q)


def _link(rng, jtype, inner, name="", extra="", full=True, tilt=True, anchor=True):
    ax = rng.normal(0, 1, 3)
    jpos = rng.uniform(-0.05, 0.05, 3) if anchor else np.zeros(3)
    q = ' quat="%s"' % _v(_quat(rng)) if tilt else ""
    return ('<body pos="%s"%s><joint %s type="%s" axis="%s" pos="%s" %s/>%s<geom type="sphere" size="0.02" %s/>'
            '<site pos="%s" quat="%s"/>%s</body>' % (_v(rng.uniform(-0.1, 0.1, 3) + [0, 0, -0.15]), q, name, jtype, _v(ax), _v(jpos), extra,
                                                     _inertial(rng, full), _OFF, _v(rng.uniform(-0.05, 0.05, 3)), _v(_quat(rng)), inner))


def hinge_chain():
    rng = np.random.default_rng(1)
    inner = ""
    for k in range(6, -1, -1):
        extra = 'armature="%.4g" damping="%.4g" ref="%.4g"' % (rng.uniform(0, 0.1), rng.uniform(0, 0.5), rng.uniform(-0.5, 0.5) * (k % 2))
        if k == 3:  # a massive dof-less body welded between two jointed links
            inner = '<body pos="0.02 0.03 -0.1" quat="%s">%s<site pos="0.01 0 0"/>%s</body>' % (_v(_quat(rng)), _inertial(rng, True, 8.0), inner)
        inner = _link(rng, "hinge", inner, extra=extra, full=k % 2 == 0)
    return _mjcf(inner)


def slide_hinge_mix():
    rng = np.random.default_rng(2)
    inner = _link(rng, "slide", "", extra='ref="-0.05" damping="0.3"')
    inner = _link(rng, "hinge", inner, extra='armature="0.02"')
    inner = _link(rng, "slide", inner, extra='ref="0.1" armature="0.05"')
    return _mjcf(inner)


def free_bodies():
    rng = np.random.default_rng(3)
    out = ""
    for k in range(3):
        child = _link(rng, "hinge", "", extra='damping="0.1"') if k == 1 else ""
        out += ('<body pos="%d 0 1" quat="%s"><freejoint/>%s<geom type="box" size="0.05 0.03 0.02" %s/><site pos="0.01 0.02 0"/>%s</body>'
                % (k, _v(_quat(rng)), _inertial(rng, True), _OFF, child))
    return _mjcf(out)


def fluid_wind():
    rng = np.random.default_rng(4)
    rod = ('<body pos="0 0 1"><freejoint/><inertial pos="0.01 0 0.02" quat="%s" mass="0.7" diaginertia="0.02 0.0201 0.00002"/>'
           '<geom type="capsule" size="0.01 0.3" %s/><site/></body>' % (_v(_quat(rng)), _OFF))
    chain = _link(rng, "hinge", _link(rng, "slide", "", full=False), extra='damping="0.05"')
    return _mjcf(rod + chain, option='density="900" viscosity="0.4" wind="1.5 -2 0.7"')


def springs():
    rng = np.random.default_rng(5)
    a = _link(rng, "hinge", "", extra='stiffness="7" ref="0.3" springref="-0.4" damping="0.1"')
    b = _link(rng, "slide", "", extra='stiffness="120" ref="0.05" springref="0.12"')
    c = _link(rng, "hinge", _link(rng, "slide", "", extra='stiffness="40" springref="-0.03"'), extra='stiffness="3" springref="0.7"')
    return _mjcf(a + b + c)


def actuators():
    rng = np.random.default_rng(6)
    body = ""
    for k in range(4):
        body += _link(rng, "hinge" if k % 2 == 0 else "slide", "", name='name="j%d"' % k, extra='damping="0.2"')
    act = ('<motor joint="j0" gear="2.5" ctrlrange="-1 1" forcerange="-1.5 1.5"/>'
           '<position joint="j1" kp="300" kv="12" gear="0.5" ctrlrange="-0.2 0.2"/>'
           '<velocity joint="j2" kv="4" gear="-1.7" forcerange="-3 3"/>'
           '<general joint="j3" gainprm="3 0 0" biasprm="0.4 -50 -2" biastype="affine" gear="1.3" ctrlrange="-2 2" forcerange="-10 8"/>')
    return _mjcf(body, actuator=act)


def gravity(g):
    rng = np.random.default_rng(7)
    chain = _link(rng, "hinge", _link(rng, "slide", _link(rng, "hinge", "")))
    free = '<body pos="1 0 1"><freejoint/>%s<geom type="sphere" size="0.03" %s/></body>' % (_inertial(rng, True), _OFF)
    return _mjcf(chain + free, option='gravity="%s"' % g)


def _chain(rng, n, welded_every=0, tip=False, full=False):
    """one tree of n dofs alternating hinge and slide joints; welded_every: a dof-less body under every k-th link"""
    inner = '<body pos="0 0 -0.05">%s<site/></body>' % _inertial(rng) if tip else ""
    for k in range(n - 1, -1, -1):
        if welded_every and k % welded_every == 0:
            inner += '<body pos="0.03 0 0">%s</body><body pos="-0.03 0 0">%s</body>' % (_inertial(rng, mass=0.1), _inertial(rng, mass=0.1))
        inner = _link(rng, "slide" if k % 3 == 1 else "hinge", inner, extra='damping="0.05" armature="0.01"', full=full and k % 4 == 0)
    return inner


# (name, tree sizes, welded bodies under every k-th link, welded tip): the largest tree picks the M-solve branch
TREE_SCENES = [
    ("tree_8", [8, 5], 0, False),      # spd_solve_blk<8>
    ("tree_9", [9, 3, 2], 0, False),   # spd_solve_blk<9>
    ("tree_12", [12, 12], 0, False),   # spd_solve_blk<12>, nv 24
    ("tree_16", [16], 0, False),       # spd_solve_reg<16>
    ("tree_24", [13, 11], 0, False),   # spd_solve_reg<24>
    ("tree_32", [32], 0, True),        # spd_solve_reg<32>, 33 levels deep
    ("chol_48", [20, 16, 12], 0, False),  # dense Cholesky
    ("chol_64", [24, 24, 16], 2, False),  # dense Cholesky at the device's nv cap, more than 64 bodies
]


def tree_scene(sizes, welded_every, tip):
    rng = np.random.default_rng(sum(sizes))
    return _mjcf("".join(_chain(rng, n, welded_every, tip, full=True) for n in sizes))


# ------------------------------------------------------------------------------------------------ states
class Case:
    """a scene, per-environment (qpos, qvel, ctrl) and optional per-environment model values (dynamics_ref.Forward's env)"""

    def __init__(self, name, model, Q, V, U, envs=None, contacts=False):
        self.name, self.model, self.Q, self.V, self.U, self.envs, self.contacts = name, model, Q, V, U, envs, contacts
        self.n = len(Q)

    def forward(self, e):
        return dr.Forward(self.model, self.Q[e], self.V[e], self.U[e], self.envs[e] if self.envs else None)


def random_states(m, n, seed, vscale=1.0, spin=0.0):
    rng = np.random.default_rng(seed)
    Q = np.tile(m.qpos0, (n, 1))
    V = rng.normal(0, vscale, (n, m.nv))
    for j in range(m.njnt):
        a, d, t = int(m.jnt_qposadr[j]), int(m.jnt_dofadr[j]), int(m.jnt_type[j])
        if t == dr.FREE:
            Q[:, a:a + 3] += rng.normal(0, 0.1, (n, 3))
            for e in range(n):
                Q[e, a + 3:a + 7] = _quat(rng)
            V[:, d + 3:d + 6] += rng.normal(0, spin, (n, 3))
        elif t == dr.HINGE:
            Q[:, a] += rng.uniform(-1.5, 1.5, n)
        else:
            Q[:, a] += rng.uniform(-0.1, 0.1, n)
    U = rng.uniform(-3, 3, (n, m.nu))
    return Q, V, U


def override_envs(m, n, seed):
    rng = np.random.default_rng(seed)
    tri = lambda I: I[0] + I[1] >= I[2] and I[0] + I[2] >= I[1] and I[1] + I[2] >= I[0]  # what the library accepts as moments
    bodies = [b for b in range(1, m.nbody) if m.body_mass[b] > 0 and tri(m.body_inertia[b])][:4]
    assert len(bodies) >= 2
    out = []
    for e in range(n):
        out.append({"body_mass": {b: float(m.body_mass[b] * rng.uniform(0.5, 2.0)) for b in bodies},
                    "body_inertia": {b: m.body_inertia[b] * rng.uniform(0.6, 1.6) for b in bodies},  # moments keep the triangle inequality
                    "dof_damping": m.dof_damping * rng.uniform(0.5, 1.5, m.nv) + rng.uniform(0, 0.3, m.nv),
                    "dof_armature": m.dof_armature * rng.uniform(0.5, 2.0, m.nv) + rng.uniform(0, 0.05, m.nv)})
    return out


PACKAGED = ["Lift_Panda", "Stack_Panda", "Door_Panda", "PickPlace_Panda", "NutAssemblyRound_Panda", "Lift_Sawyer"]


def packaged_case(name, n, seed):
    """a packaged model at seeded states: arm near its home pose, objects in place, the Door's latch turned"""
    from tests.util import PANDA_INIT, load

    m = load(name)
    rng = np.random.default_rng(seed)
    Q = np.tile(m.qpos0, (n, 1))
    arm = [j for j, nm in enumerate(m.names["joint"]) if nm and nm.startswith("robot0_") and int(m.jnt_type[j]) == dr.HINGE]
    for k, j in enumerate(arm[:7]):
        Q[:, int(m.jnt_qposadr[j])] = (PANDA_INIT[k] if name.endswith("Panda") else 0.3 * np.sin(k)) + rng.normal(0, 0.05, n)
    latch = m.name2id("joint", "Door_latch_joint")
    if latch >= 0:
        Q[:, int(m.jnt_qposadr[latch])] = rng.uniform(0.3, 1.2, n)
    V = rng.normal(0, 0.3, (n, m.nv))
    U = rng.uniform(-1, 1, (n, m.nu))
    return Case(name, m, Q, V, U, contacts=True)


def catalogue(n=4, seed=0, packaged=True):
    out = []

    def add(name, xml, vscale=1.0, spin=0.0, envs=False):
        m = compile_scene(xml)
        Q, V, U = random_states(m, n, seed + len(out), vscale, spin)
        out.append(Case(name, m, Q, V, U, override_envs(m, n, seed + 50 + len(out)) if envs else None))

    add("hinge_chain", hinge_chain())
    add("slide_hinge_mix", slide_hinge_mix())
    add("free_bodies", free_bodies(), spin=3.0)
    add("fluid_wind", fluid_wind(), vscale=3.0, spin=10.0)
    add("springs", springs())
    add("actuators", actuators())
    add("gravity_tilted", gravity("3 -4 -8"))
    add("gravity_zero", gravity("0 0 0"))
    for name, sizes, we, tip in TREE_SCENES:
        add(name, tree_scene(sizes, we, tip), vscale=0.5)
    add("overrides", hinge_chain(), envs=True)
    if packaged:
        for k, name in enumerate(PACKAGED):
            out.append(packaged_case(name, min(n, 3), seed + 100 + k))
    return out


_CAT = {}


def cached_catalogue(**kw):
    key = tuple(sorted(kw.items()))
    if key not in _CAT:
        _CAT[key] = catalogue(**kw)
    return _CAT[key]


SCENES = (["hinge_chain", "slide_hinge_mix", "free_bodies", "fluid_wind", "springs", "actuators", "gravity_tilted", "gravity_zero"]
          + [t[0] for t in TREE_SCENES] + ["overrides"])
CASE_NAMES = SCENES + PACKAGED


def case_named(name, **kw):
    return next(c for c in cached_catalogue(**kw) if c.name == name)


def rel_err(a, b):
    """largest |a - b| relative to |b| plus the array's own scale"""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    if a.size == 0:
        return 0.0
    return float((np.abs(a - b) / (np.abs(b) + np.abs(b).max() + 1e-300)).max())


def quat_err(a, b):
    """rel_err of unit quaternions up to sign, row by row"""
    a, b = np.asarray(a, dtype=np.float64).reshape(-1, 4), np.asarray(b, dtype=np.float64).reshape(-1, 4)
    s = np.where(np.sum(a * b, axis=1) < 0, -1.0, 1.0)[:, None]
    return rel_err(a * s, b)


def model_of(case, e):
    """the model with environment e's values written in (what the oracle runs)"""
    import copy

    if not case.envs:
        return case.model
    m = copy.deepcopy(case.model)
    v = case.envs[e]
    for b, x in v["body_mass"].items():
        m.body_mass[b] = x
    for b, x in v["body_inertia"].items():
        m.body_inertia[b] = x
    m.dof_damping, m.dof_armature = np.array(v["dof_damping"]), np.array(v["dof_armature"])
    return m


def oracle_forward(m, q, v, u):
    from oracle.pyoracle import Oracle
    from robosuite_b200.mjcf.compiler import pack_model

    o = Oracle(pack_model(m))
    o.reset_data()
    o.qpos[:], o.qvel[:], o.ctrl[:] = q, v, u
    o.forward()
    return o


# ------------------------------------------------------------------------------------------------ the reference itself
def _fd_case_states():
    for name in ["hinge_chain", "slide_hinge_mix", "free_bodies", "fluid_wind", "tree_9"]:
        c = case_named(name, packaged=False)
        yield c, c.Q[0], c.V[0]


def perturb(m, q, d, eps):
    """q displaced by eps along dof d (free rotations in body axes)"""
    q = q.copy()
    j = int(m.dof_jntid[d])
    a, k = int(m.jnt_qposadr[j]), d - int(m.jnt_dofadr[j])
    if int(m.jnt_type[j]) == dr.FREE and k >= 3:
        w = np.zeros(3)
        w[k - 3] = 1
        r = dr.qmul(q[a + 3:a + 7], dr.qexp(w, eps))
        q[a + 3:a + 7] = r
    elif int(m.jnt_type[j]) == dr.FREE:
        q[a + k] += eps
    else:
        q[a] += eps
    return q


def _rotvec(R):
    from scipy.spatial.transform import Rotation

    return Rotation.from_matrix(R).as_rotvec()


def test_jacobians_match_differenced_kinematics():
    eps = 1e-6
    for c, q, _ in _fd_case_states():
        m = c.model
        k = dr.Kin(m, q)
        for b in range(1, m.nbody):
            Jp, Jr = k.jac(b, k.xipos[b])
            for d in range(m.nv):
                kp, km = dr.Kin(m, perturb(m, q, d, eps)), dr.Kin(m, perturb(m, q, d, -eps))
                dp = (kp.xipos[b] - km.xipos[b]) / (2 * eps)
                dw = _rotvec(kp.ximat[b] @ km.ximat[b].T) / (2 * eps)
                assert np.allclose(dp, Jp[:, d], atol=1e-8, rtol=1e-6), (c.name, b, d, dp, Jp[:, d])
                assert np.allclose(dw, Jr[:, d], atol=1e-8, rtol=1e-6), (c.name, b, d, dw, Jr[:, d])


def test_mass_matrix_is_the_sum_of_body_jacobians():
    for c, q, _ in _fd_case_states():
        m = c.model
        k = dr.Kin(m, q)
        M = dr.mass_matrix(m, k)
        S = np.diag(np.asarray(m.dof_armature, dtype=np.float64))
        for b in range(1, m.nbody):
            Jp, Jr = k.jac(b, k.xipos[b])
            Iw = k.ximat[b] @ np.diag(m.body_inertia[b]) @ k.ximat[b].T
            S += m.body_mass[b] * Jp.T @ Jp + Jr.T @ Iw @ Jr
        assert rel_err(M, S) < 1e-13, c.name
        assert np.abs(M - M.T).max() <= 1e-13 * np.abs(M).max()
        assert np.linalg.eigvalsh(M).min() > 0


def test_kinetic_energy_from_differenced_body_velocities():
    eps = 1e-6
    for c, q, qd in _fd_case_states():
        m = c.model
        k = dr.Kin(m, q)
        M = dr.mass_matrix(m, k, armature=np.zeros(m.nv))
        h = eps
        kp, km = dr.Kin(m, dr.integrate(m, q, qd, h)[0]), dr.Kin(m, dr.integrate(m, q, -qd, h)[0])
        T = 0.0
        for b in range(1, m.nbody):
            vc = (kp.xipos[b] - km.xipos[b]) / (2 * h)
            w = _rotvec(kp.ximat[b] @ km.ximat[b].T) / (2 * h)
            Iw = k.ximat[b] @ np.diag(m.body_inertia[b]) @ k.ximat[b].T
            T += 0.5 * m.body_mass[b] * vc @ vc + 0.5 * w @ Iw @ w
        assert T == pytest.approx(0.5 * qd @ M @ qd, rel=1e-7), c.name


def test_bias_is_the_lagrangian_on_scalar_joints():
    """qfrc_bias = dM/dt qd - d/dq (qd M qd / 2) + dV/dq, dM/dq by central differences"""
    eps = 1e-6
    for name in ["hinge_chain", "slide_hinge_mix", "tree_9", "gravity_tilted"]:
        c = case_named(name, packaged=False)
        m = c.model
        if any(int(t) == dr.FREE for t in m.jnt_type):
            continue
        q, qd = c.Q[1], c.V[1]
        g = np.asarray(m.opt_gravity, dtype=np.float64)
        Mq = lambda x: dr.mass_matrix(m, dr.Kin(m, x), armature=np.zeros(m.nv))
        V = lambda x: -sum(m.body_mass[b] * g @ dr.Kin(m, x).xipos[b] for b in range(1, m.nbody))
        dM = [(Mq(q + eps * np.eye(m.nv)[i]) - Mq(q - eps * np.eye(m.nv)[i])) / (2 * eps) for i in range(m.nv)]
        Mdot = sum(dM[i] * qd[i] for i in range(m.nv))
        lag = Mdot @ qd - np.array([0.5 * qd @ dM[i] @ qd for i in range(m.nv)])
        lag += np.array([(V(q + eps * np.eye(m.nv)[i]) - V(q - eps * np.eye(m.nv)[i])) / (2 * eps) for i in range(m.nv)])
        bias = dr.rnea(m, dr.Kin(m, q), qd, np.zeros(m.nv), g)
        assert np.allclose(bias, lag, rtol=1e-6, atol=1e-6 * np.abs(lag).max()), (name, bias, lag)


@pytest.mark.parametrize("ipos", ["0 0 0", "0.05 -0.02 0.03"])
def test_bias_of_a_lone_free_body_closed_form(ipos):
    m = compile_scene(_mjcf('<body pos="0 0 1"><freejoint/><inertial pos="%s" quat="0.9 0.1 -0.3 0.2" mass="1.7" '
                            'diaginertia="0.03 0.02 0.01"/></body>' % ipos, option='gravity="0.5 -1 -9.81"'))
    rng = np.random.default_rng(0)
    q = np.r_[rng.normal(0, 1, 3), _quat(rng)]
    qd = rng.normal(0, 3, 6)
    k = dr.Kin(m, q)
    R, c, mass = k.xmat[1], np.asarray(m.body_ipos[1], dtype=np.float64), float(m.body_mass[1])
    Ri = dr.quat2mat(m.body_iquat[1])
    Ic = Ri @ np.diag(m.body_inertia[1]) @ Ri.T  # about the com, body axes
    w, g = qd[3:], np.asarray(m.opt_gravity, dtype=np.float64)
    # zero generalised acceleration: the origin does not accelerate and w is constant, so the com accelerates by R (w x (w x c))
    F = mass * (R @ np.cross(w, np.cross(w, c)) - g)  # world force on the origin's translation dofs
    exp = np.r_[F, np.cross(w, Ic @ w) + np.cross(c, R.T @ F)]  # body-axes torque about the origin on the rotation dofs
    bias = dr.rnea(m, k, qd, np.zeros(6), g)
    assert np.allclose(bias, exp, rtol=1e-12, atol=1e-12 * np.abs(exp).max()), (bias, exp)


def test_fluid_and_wind_at_hand_set_velocities():
    m = compile_scene(_mjcf('<body pos="0 0 1"><freejoint/><inertial pos="0 0 0" mass="2" diaginertia="0.05 0.04 0.03"/></body>',
                            option='density="1000" viscosity="0.2" wind="1 2 -1"'))
    q = np.r_[0, 0, 1, 1, 0, 0, 0.0]
    qd = np.array([3.0, -1.0, 0.5, 0.4, -2.0, 1.0])
    I, mass = np.array([0.05, 0.04, 0.03]), 2.0
    box = np.sqrt(np.array([I[1] + I[2] - I[0], I[0] + I[2] - I[1], I[0] + I[1] - I[2]]) / mass * 6)
    d = box.mean()
    v = qd[:3] - np.array([1, 2, -1.0])
    w = qd[3:]
    F = -3 * np.pi * d * 0.2 * v - 0.5 * 1000 * np.array([box[1] * box[2], box[0] * box[2], box[0] * box[1]]) * np.abs(v) * v
    Tq = -np.pi * d ** 3 * 0.2 * w - 1000 * box * np.array([box[1] ** 4 + box[2] ** 4, box[0] ** 4 + box[2] ** 4,
                                                             box[0] ** 4 + box[1] ** 4]) * np.abs(w) * w / 64
    f = dr.Forward(m, q, qd)
    assert np.allclose(f.qfrc_fluid, np.r_[F, Tq], rtol=1e-13, atol=0)
    assert np.allclose(f.qfrc_passive, np.r_[F, Tq], rtol=1e-13, atol=0)


def test_springs_closed_form():
    c = case_named("springs", packaged=False)
    m = c.model
    assert np.any(m.qpos_spring != m.qpos0)
    f = dr.Forward(m, c.Q[0], c.V[0])
    exp = -np.asarray(m.dof_damping) * c.V[0]
    for j in range(m.njnt):
        a = int(m.jnt_qposadr[j])
        exp[int(m.jnt_dofadr[j])] -= m.jnt_stiffness[j] * (c.Q[0][a] - m.qpos_spring[a])
    assert np.allclose(f.qfrc_spring_damper, exp, rtol=1e-15, atol=0)


def test_euler_free_rotation_known_answer():
    m = compile_scene(_mjcf('<body pos="0 0 0"><freejoint/><inertial pos="0 0 0" mass="1" diaginertia="0.1 0.1 0.1"/></body>',
                            option='gravity="0 0 0"'))
    rng = np.random.default_rng(1)
    q0 = np.r_[0, 0, 0, _quat(rng)]
    w = np.array([3.0, -7.0, 11.0])
    q, qd = q0.copy(), np.r_[0, 0, 0, w]
    n = 50
    for _ in range(n):
        f = dr.Forward(m, q, qd)
        assert np.allclose(f.qacc_smooth, 0, atol=1e-12)
        q, qd = f.euler()
    exp = dr.qmul(q0[3:], dr.qexp(w, n * float(m.opt_timestep)))
    assert np.abs(q[3:] - exp).max() < 1e-13


def test_euler_damped_slide_closed_form():
    m = compile_scene(_mjcf('<body><joint type="slide" axis="0 0 1" damping="30"/><inertial pos="0 0 0" mass="0.5" '
                            'diaginertia="0.01 0.01 0.01"/></body>', option='gravity="0 0 -9.81"'))
    h, mass, b = 0.002, 0.5, 30.0
    q, v = np.array([0.1]), np.array([2.0])
    f = dr.Forward(m, q, v)
    q1, v1 = f.euler()
    a = (-b * v[0] - mass * 9.81) / (mass + h * b)
    assert v1[0] == pytest.approx(v[0] + h * a, rel=1e-14)
    assert q1[0] == pytest.approx(q[0] + h * v1[0], rel=1e-14)


# ------------------------------------------------------------------------------------------------ the catalogue's reach
def test_catalogue_reaches_every_m_solve_branch():
    """the device picks spd_solve_blk<8|9|12> by the largest tree when nv <= 32, spd_solve_reg<16|24|32> by nv otherwise, and the
    dense Cholesky above 32"""
    def branch(m):
        nv, ts = dr.trees(m)
        if nv <= 32 and ts <= 12:
            return "blk%d" % (8 if ts <= 8 else 9 if ts <= 9 else 12)
        if nv <= 32:
            return "reg%d" % (16 if nv <= 16 else 24 if nv <= 24 else 32)
        return "chol"
    got = {c.name: branch(c.model) for c in cached_catalogue(packaged=False)}
    for name, want in [("tree_8", "blk8"), ("tree_9", "blk9"), ("tree_12", "blk12"), ("tree_16", "reg16"), ("tree_24", "reg24"),
                       ("tree_32", "reg32"), ("chol_48", "chol"), ("chol_64", "chol")]:
        assert got[name] == want, (name, got[name])
    m64 = case_named("chol_64", packaged=False).model
    assert m64.nv == 64 and m64.nbody > 65
    depth = lambda m, b: 0 if b == 0 else 1 + depth(m, int(m.body_parentid[b]))
    m32 = case_named("tree_32", packaged=False).model
    assert max(depth(m32, b) for b in range(m32.nbody)) > 32


GPU_CAPACITY = (2, 8)  # (maxcon, maxefc) the device tests give the contact-free scenes


def test_catalogue_scenes_fit_shared_memory():
    import ctypes as C

    from tests.test_cpu_layouts import _lib

    L = _lib()
    for c in cached_catalogue(packaged=False):
        m = c.model
        words = (C.c_int * 5)()
        mc, me = GPU_CAPACITY
        assert L.b2s_debug_layouts(m.nq, m.nv, m.nu, m.nbody, 0, m.nsite, 1, mc, me, mc, me, 0, words, None, None) == 0
        for rsz in (4, 8):
            assert max(words) * rsz <= 226 * 1024, (c.name, rsz, list(words))


def test_compiler_rejects_unsupported_dynamics():
    from robosuite_b200.mjcf.compiler import compile_mjcf

    body = '<body><joint type="hinge" name="j"/><inertial pos="0 0 0" mass="1" diaginertia="1 1 1"/></body>'
    bad = [
        _mjcf('<body gravcomp="1"><joint type="hinge"/><inertial pos="0 0 0" mass="1" diaginertia="1 1 1"/></body>'),
        _mjcf('<body><joint type="hinge" springdamper="0.1 0.5"/><inertial pos="0 0 0" mass="1" diaginertia="1 1 1"/></body>'),
        _mjcf('<body><freejoint/><joint type="free" stiffness="2"/><inertial pos="0 0 0" mass="1" diaginertia="1 1 1"/></body>'
              .replace("<freejoint/>", "")),
        _mjcf(body, actuator='<general joint="j" dyntype="filter"/>'),
        _mjcf(body, actuator='<general joint="j" gaintype="affine"/>'),
        _mjcf(body, actuator='<general joint="j" biastype="muscle"/>'),
    ]
    for xml in bad:
        with pytest.raises(NotImplementedError):
            compile_mjcf(xml)
    compile_mjcf(_mjcf(body, actuator='<general joint="j" dyntype="none" gaintype="fixed" biastype="affine"/>'))
    compile_mjcf(_mjcf('<body><joint type="hinge" springdamper="0 0"/><inertial pos="0 0 0" mass="1" diaginertia="1 1 1"/></body>'))


def test_packaged_xmls_compile_with_spring_references(monkeypatch):
    """the seven packaged MJCF files pass the new rejections; their meshes (not in the tree) are stood in for by a tetrahedron"""
    import glob
    import os

    from robosuite_b200.mjcf import meshio
    from robosuite_b200.mjcf.compiler import compile_mjcf, load_model
    from tests.util import ROOT, load

    tet = (np.array([[0, 0, 0], [0.01, 0, 0], [0, 0.01, 0], [0, 0, 0.01]], dtype=np.float64),
           np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]]))
    monkeypatch.setattr(meshio, "load_mesh", lambda path: (tet[0].copy(), tet[1].copy()))

    files = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "mjcf", "*.xml")))
    assert len(files) == 7
    for f in files:
        with open(f) as fh:
            m = compile_mjcf(fh.read(), mesh_root=os.path.dirname(f))
        name = os.path.basename(f)[:-4]
        fixture = load(name)
        asset = load_model(os.path.join(ROOT, "robosuite_b200", "assets", "models", name + ".npz"))  # stored without qpos_spring
        for x in (m, fixture, asset):
            assert np.array_equal(x.qpos_spring, x.qpos0), f


def test_spring_reference_and_hinge_angles_in_degrees():
    from robosuite_b200.mjcf.compiler import compile_mjcf

    m = compile_mjcf('<mujoco><worldbody><body><joint type="hinge" ref="30" springref="-45" stiffness="1"/><inertial pos="0 0 0" '
                     'mass="1" diaginertia="1 1 1"/></body><body><joint type="slide" ref="0.2" springref="0.3"/><inertial pos="0 0 0" '
                     'mass="1" diaginertia="1 1 1"/></body><body><freejoint/><inertial pos="0 0 0" mass="1" diaginertia="1 1 1"/></body>'
                     '</worldbody></mujoco>')
    assert np.allclose(m.qpos0[:2], [np.pi / 6, 0.2]) and np.allclose(m.qpos_spring[:2], [-np.pi / 4, 0.3])
    assert np.array_equal(m.qpos_spring[2:], m.qpos0[2:])


# ------------------------------------------------------------------------------------------------ the oracle against the reference
ORACLE_FIELDS = ["xpos", "xmat", "site_xpos", "site_xmat", "cdof", "M", "qfrc_bias", "qfrc_passive", "qfrc_actuator", "actuator_force",
                 "qfrc_smooth", "qacc_smooth"]


def compare_forward(f, get, quat=None):
    """{field: rel_err} of an engine's forward outputs (get(field) -> array) against the reference f.  qacc_smooth is judged by its
    residual M a - qfrc_smooth against the reference's M and force: near-rod inertias make M ill-conditioned, and the error of a
    backward-stable solve is bounded in force, not in acceleration"""
    out = {}
    for k in ORACLE_FIELDS:
        ref = getattr(f, k)
        if np.size(ref) == 0:
            continue
        a = np.asarray(get(k), dtype=np.float64).reshape(np.shape(ref))
        out[k] = rel_err(f.M @ a, f.qfrc_smooth) if k == "qacc_smooth" else rel_err(a, ref)
    if quat is not None:
        out["xquat"] = quat_err(quat, f.xquat)
    return out


def step_errors(f, q1, v1):
    """errors of an engine's Euler step (q1, v1) from the reference state f: the velocity update by its residual
    (M + h D) (v1 - qvel) / h - qfrc_smooth (as compare_forward judges qacc_smooth), the position update against the reference's
    integration of v1"""
    m, h = f.m, float(f.m.opt_timestep)
    q1, v1 = np.asarray(q1, dtype=np.float64), np.asarray(v1, dtype=np.float64)
    A = f.M + h * np.diag(f.damping)
    return {"qvel_residual": rel_err(A @ (v1 - f.qd) / h, f.qfrc_smooth), "qpos_of_qvel": rel_err(q1, dr.integrate(m, f.q, v1, h)[0])}


@pytest.mark.parametrize("name", CASE_NAMES)
def test_oracle_matches_reference(name):
    c = case_named(name)
    for e in range(c.n):
        f = c.forward(e)
        o = oracle_forward(model_of(c, e), c.Q[e], c.V[e], c.U[e])
        errs = compare_forward(f, lambda k: getattr(o, k), o.xquat)
        bad = {k: v for k, v in errs.items() if not v <= ORACLE_RTOL}
        assert not bad, (name, e, bad)
        if not c.contacts:
            o2 = oracle_forward(model_of(c, e), c.Q[e], c.V[e], c.U[e])
            o2.step()
            errs = step_errors(f, o2.qpos, o2.qvel)
            assert max(errs.values()) <= ORACLE_RTOL, (name, e, errs)
