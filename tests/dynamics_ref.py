"""An independent fp64 statement of the engine's smooth dynamics, for test_cpu_dynamics.py and test_gpu_dynamics.py.

Written from the engine's documented definitions, not from the oracle's or the device's code, and organised differently on purpose:
the device and the oracle work with world-origin spatial algebra and 10-number inertias; this file works with 4x4 homogeneous
transforms, Featherstone's recursive Newton-Euler in body-local coordinates (6x6 Plucker transforms, each joint's motion subspace
in its own body's frame) and Jacobians formed from the homogeneous kinematics.

- Kinematics: T_body = T_parent . T(body_pos, body_quat) . T_joint.  A hinge rotates about its anchor jnt_pos by q - qpos0, a slide
  translates along its axis by q - qpos0, a free joint gives the world pose from qpos.  Inertial, geom and site frames follow from
  the body's transform and their local (pos, quat).
- Free-joint velocity convention: linear velocity of the body origin in world axes, angular velocity in body axes.
- qfrc_bias = RNEA(q, qd, 0) with gravity as base acceleration; M = columns RNEA(q, 0, e_k) without gravity, plus diag(armature).
- Passive force: -damping qd; -stiffness (q - qpos_spring) on hinge and slide joints; the inertia-box fluid model (the body's
  inertial-frame velocity with the wind subtracted, viscous and quadratic terms) mapped back through the Jacobian at xipos.
- Actuation: force = gain ctrl + (affine bias on length q gear and velocity qd gear), ctrl and force clamps; moment gear force.
- Euler: (M + h diag(damping)) a = qfrc_smooth + qfrc_constraint; qd += h a; hinge / slide q += h qd; free pos += h v and
  quat <- quat (x) exp(h w / 2) (body axes), normalised.
"""
import numpy as np
from scipy.spatial.transform import Rotation

FREE, BALL, SLIDE, HINGE = 0, 1, 2, 3
MINVAL = 1e-15


# ------------------------------------------------------------------------------------------------ small algebra
def quat2mat(q):
    q = np.asarray(q, dtype=np.float64)
    return Rotation.from_quat([q[1], q[2], q[3], q[0]]).as_matrix()


def mat2quat(R):
    x, y, z, w = Rotation.from_matrix(R).as_quat()
    return np.array([w, x, y, z])


def qmul(a, b):
    w1, x1, y1, z1 = a
    w2, x2, y2, z2 = b
    return np.array([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                     w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2])


def qexp(w, t):
    """the unit quaternion of a rotation by |w| t about w"""
    n = np.linalg.norm(w)
    if n < MINVAL:
        return np.array([1.0, 0, 0, 0])
    a = n * t
    return np.r_[np.cos(a / 2), np.sin(a / 2) * np.asarray(w) / n]


def hom(p, R):
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, p
    return T


def skew(v):
    return np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]])


def plucker(T):
    """motion-vector transform from a parent frame to a child frame whose pose in the parent is T: [w; v] -> child coordinates"""
    E, p = T[:3, :3].T, T[:3, 3]
    X = np.zeros((6, 6))
    X[:3, :3] = E
    X[3:, 3:] = E
    X[3:, :3] = -E @ skew(p)
    return X


def crm(v):
    """v x (motion)"""
    X = np.zeros((6, 6))
    X[:3, :3] = skew(v[:3])
    X[3:, 3:] = skew(v[:3])
    X[3:, :3] = skew(v[3:])
    return X


def crf(v):
    """v x* (force)"""
    return -crm(v).T


# ------------------------------------------------------------------------------------------------ model views
def chain_dofs(m, b):
    """dofs on the kinematic chain from the world to body b"""
    out = []
    while b > 0:
        for d in range(int(m.body_dofadr[b]), int(m.body_dofadr[b]) + int(m.body_dofnum[b])):
            out.append(d)
        b = int(m.body_parentid[b])
    return sorted(out)


def body_joint(m, b):
    n = int(m.body_jntnum[b])
    assert n <= 1, "one joint per body"
    return int(m.body_jntadr[b]) if n else -1


def qpos_spring(m):
    return np.asarray(getattr(m, "qpos_spring", m.qpos0), dtype=np.float64)


def trees(m):
    """(nv, size of the largest kinematic tree in dofs)"""
    sizes = {}
    for d in range(m.nv):
        b = int(m.dof_bodyid[d])
        while int(m.body_parentid[b]) != 0:
            b = int(m.body_parentid[b])
        sizes[b] = sizes.get(b, 0) + 1
    return int(m.nv), max(sizes.values()) if sizes else 0


# ------------------------------------------------------------------------------------------------ kinematics
class Kin:
    """homogeneous kinematics of one state: body, inertial, geom and site transforms, joint anchors and axes"""

    def __init__(self, m, q, body_pose=None):
        self.m = m
        nb = int(m.nbody)
        q0 = np.asarray(m.qpos0, dtype=np.float64)
        self.T = [np.eye(4) for _ in range(nb)]
        self.Tloc = [np.eye(4) for _ in range(nb)]  # body frame in its parent's frame, joint displacement included
        self.anchor = np.zeros((int(m.njnt), 3))
        self.axis = np.zeros((int(m.njnt), 3))
        for b in range(1, nb):
            pos, quat = np.asarray(m.body_pos[b], dtype=np.float64), np.asarray(m.body_quat[b], dtype=np.float64)
            if body_pose is not None and b in body_pose:
                pos, quat = body_pose[b]
            Tl = hom(pos, quat2mat(quat))
            j = body_joint(m, b)
            par = int(m.body_parentid[b])
            if j >= 0:
                a, t = int(m.jnt_qposadr[j]), int(m.jnt_type[j])
                ax, jp = np.asarray(m.jnt_axis[j], dtype=np.float64), np.asarray(m.jnt_pos[j], dtype=np.float64)
                if t == FREE:
                    qq = q[a + 3:a + 7] / np.linalg.norm(q[a + 3:a + 7])
                    Tw = hom(q[a:a + 3], quat2mat(qq))
                    Tl = np.linalg.inv(self.T[par]) @ Tw
                elif t == SLIDE:
                    Tl = Tl @ hom(ax * (q[a] - q0[a]), np.eye(3))
                elif t == HINGE:
                    Rj = Rotation.from_rotvec(ax * (q[a] - q0[a])).as_matrix()
                    Tl = Tl @ hom(jp, np.eye(3)) @ hom(np.zeros(3), Rj) @ hom(-jp, np.eye(3))
                else:
                    raise NotImplementedError("ball joints")
            self.Tloc[b] = Tl
            self.T[b] = self.T[par] @ Tl
            if j >= 0 and int(m.jnt_type[j]) != FREE:
                self.anchor[j] = self.T[b][:3, :3] @ m.jnt_pos[j] + self.T[b][:3, 3]
                self.axis[j] = self.T[b][:3, :3] @ m.jnt_axis[j]
        self.xpos = np.array([T[:3, 3] for T in self.T])
        self.xmat = np.array([T[:3, :3] for T in self.T])
        self.Ti = [self.T[b] @ hom(m.body_ipos[b], quat2mat(m.body_iquat[b])) for b in range(nb)]
        self.xipos = np.array([T[:3, 3] for T in self.Ti])
        self.ximat = np.array([T[:3, :3] for T in self.Ti])
        self.geom = [self.T[int(m.geom_bodyid[g])] @ hom(m.geom_pos[g], quat2mat(m.geom_quat[g])) for g in range(int(m.ngeom))]
        self.site = [self.T[int(m.site_bodyid[s])] @ hom(m.site_pos[s], quat2mat(m.site_quat[s])) for s in range(int(m.nsite))]

    def dof_axes(self):
        """per dof: (angular axis or None, linear direction or None, point on the axis) in world coordinates"""
        m, out = self.m, []
        for d in range(int(m.nv)):
            j = int(m.dof_jntid[d])
            b, t, k = int(m.jnt_bodyid[j]), int(m.jnt_type[j]), d - int(m.jnt_dofadr[j])
            if t == FREE:
                out.append((None, np.eye(3)[k], None) if k < 3 else (self.xmat[b][:, k - 3], None, self.xpos[b]))
            elif t == SLIDE:
                out.append((None, self.axis[j], None))
            else:
                out.append((self.axis[j], None, self.anchor[j]))
        return out

    def cdof(self):
        """world-origin motion axes [w; velocity of the point at the world origin]"""
        out = np.zeros((int(self.m.nv), 6))
        for d, (w, v, p) in enumerate(self.dof_axes()):
            out[d] = np.r_[np.zeros(3), v] if w is None else np.r_[w, np.cross(p, w)]
        return out

    def jac(self, b, point):
        """(3 x nv translational, 3 x nv rotational) Jacobian of a world point attached to body b"""
        m = self.m
        Jp, Jr = np.zeros((3, int(m.nv))), np.zeros((3, int(m.nv)))
        axes = self.dof_axes()
        for d in chain_dofs(m, b):
            w, v, p = axes[d]
            if w is None:
                Jp[:, d] = v
            else:
                Jr[:, d] = w
                Jp[:, d] = np.cross(w, point - p)
        return Jp, Jr


# ------------------------------------------------------------------------------------------------ dynamics
def body_inertia6(m, b, mass=None, inertia=None):
    """6x6 spatial inertia of body b about its origin in body coordinates"""
    mass = float(m.body_mass[b] if mass is None else mass)
    inertia = np.asarray(m.body_inertia[b] if inertia is None else inertia, dtype=np.float64)
    Ri = quat2mat(m.body_iquat[b])
    Ic = Ri @ np.diag(inertia) @ Ri.T
    c = np.asarray(m.body_ipos[b], dtype=np.float64)
    C = skew(c)
    I = np.zeros((6, 6))
    I[:3, :3] = Ic + mass * C @ C.T
    I[:3, 3:] = mass * C
    I[3:, :3] = mass * C.T
    I[3:, 3:] = mass * np.eye(3)
    return I


def subspace(m, kin, b):
    """(joint, motion subspace 6 x ndof in body b's coordinates)"""
    j = body_joint(m, b)
    if j < 0:
        return -1, np.zeros((6, 0))
    t = int(m.jnt_type[j])
    ax, jp = np.asarray(m.jnt_axis[j], dtype=np.float64), np.asarray(m.jnt_pos[j], dtype=np.float64)
    if t == FREE:
        S = np.zeros((6, 6))
        S[3:, :3] = kin.xmat[b].T  # world-axes linear velocity of the origin, seen in body axes
        S[:3, 3:] = np.eye(3)
        return j, S
    if t == SLIDE:
        return j, np.r_[np.zeros(3), ax].reshape(6, 1)
    return j, np.r_[ax, np.cross(jp, ax)].reshape(6, 1)


def rnea(m, kin, qd, qdd, gravity, body=None):
    """generalised forces of (qd, qdd) at kin's pose; gravity: the 3-vector entering as base acceleration -g.  body: per-body
    (mass, inertia) overrides {b: (mass, inertia3)}"""
    nb, nv = int(m.nbody), int(m.nv)
    v = [np.zeros(6) for _ in range(nb)]
    a = [np.zeros(6) for _ in range(nb)]
    a[0] = np.r_[np.zeros(3), -np.asarray(gravity, dtype=np.float64)]
    f = [np.zeros(6) for _ in range(nb)]
    X = [None] * nb
    Sj = [None] * nb
    for b in range(1, nb):
        par = int(m.body_parentid[b])
        X[b] = plucker(kin.Tloc[b])
        j, S = subspace(m, kin, b)
        Sj[b] = (j, S)
        vp, ap = X[b] @ v[par], X[b] @ a[par]
        if j >= 0:
            da = int(m.jnt_dofadr[j])
            n = S.shape[1]
            vJ = S @ qd[da:da + n]
            v[b] = vp + vJ
            a[b] = ap + S @ qdd[da:da + n] + crm(v[b]) @ vJ
            if int(m.jnt_type[j]) == FREE:  # S's translation columns turn with the body: dS/dt qd = [0; -w x (R^T v_world)]
                w = qd[da + 3:da + 6]
                a[b] = ap + S @ qdd[da:da + n] + np.r_[np.zeros(3), -np.cross(w, kin.xmat[b].T @ qd[da:da + 3])]
        else:
            v[b], a[b] = vp, ap
        mb, ib = (body or {}).get(b, (None, None))
        I = body_inertia6(m, b, mb, ib)
        f[b] = I @ a[b] + crf(v[b]) @ I @ v[b]
    tau = np.zeros(nv)
    for b in range(nb - 1, 0, -1):
        j, S = Sj[b]
        if j >= 0:
            da = int(m.jnt_dofadr[j])
            tau[da:da + S.shape[1]] = S.T @ f[b]
        par = int(m.body_parentid[b])
        if par > 0:
            f[par] = f[par] + X[b].T @ f[b]
    return tau


def mass_matrix(m, kin, armature=None, body=None):
    nv = int(m.nv)
    M = np.zeros((nv, nv))
    z = np.zeros(nv)
    for k in range(nv):
        M[:, k] = rnea(m, kin, z, np.eye(nv)[k], np.zeros(3), body)
    arm = np.asarray(m.dof_armature if armature is None else armature, dtype=np.float64)
    return M + np.diag(arm)


def fluid_force(m, kin, b, qd, mass=None, inertia=None):
    """(world force, world torque) of the inertia-box fluid model on body b, acting at xipos"""
    mass = float(m.body_mass[b] if mass is None else mass)
    I = np.asarray(m.body_inertia[b] if inertia is None else inertia, dtype=np.float64)
    rho, mu = float(m.opt_density), float(m.opt_viscosity)
    if mass < MINVAL or (rho <= 0 and mu <= 0):
        return np.zeros(3), np.zeros(3)
    box = np.sqrt(np.maximum(MINVAL, np.array([I[1] + I[2] - I[0], I[0] + I[2] - I[1], I[0] + I[1] - I[2]])) / mass * 6.0)
    Jp, Jr = kin.jac(b, kin.xipos[b])
    Ri = kin.ximat[b]
    w = Ri.T @ (Jr @ qd)
    vl = Ri.T @ (Jp @ qd - np.asarray(getattr(m, "opt_wind", np.zeros(3)), dtype=np.float64))
    tq, fr = np.zeros(3), np.zeros(3)
    if mu > 0:
        d = box.mean()
        tq += -np.pi * d ** 3 * mu * w
        fr += -3 * np.pi * d * mu * vl
    if rho > 0:
        area = np.array([box[1] * box[2], box[0] * box[2], box[0] * box[1]])
        fr += -0.5 * rho * area * np.abs(vl) * vl
        b4 = box ** 4
        tq += -rho * box * np.array([b4[1] + b4[2], b4[0] + b4[2], b4[0] + b4[1]]) * np.abs(w) * w / 64.0
    return Ri @ fr, Ri @ tq


def passive(m, kin, q, qd, damping=None, body=None):
    """(total, damping + spring part, fluid part)"""
    damping = np.asarray(m.dof_damping if damping is None else damping, dtype=np.float64)
    p = -damping * qd
    qs = qpos_spring(m)
    for j in range(int(m.njnt)):
        if int(m.jnt_type[j]) in (SLIDE, HINGE):
            a = int(m.jnt_qposadr[j])
            p[int(m.jnt_dofadr[j])] -= float(m.jnt_stiffness[j]) * (q[a] - qs[a])
    fl = np.zeros(int(m.nv))
    for b in range(1, int(m.nbody)):
        mb, ib = (body or {}).get(b, (None, None))
        F, Tq = fluid_force(m, kin, b, qd, mb, ib)
        if np.any(F) or np.any(Tq):
            Jp, Jr = kin.jac(b, kin.xipos[b])
            fl += Jp.T @ F + Jr.T @ Tq
    return p + fl, p, fl


def actuation(m, q, qd, ctrl):
    """(qfrc_actuator, actuator_force)"""
    nu = int(m.nu)
    force = np.zeros(nu)
    qf = np.zeros(int(m.nv))
    for i in range(nu):
        c = float(ctrl[i])
        if m.actuator_ctrllimited[i]:
            c = min(max(c, m.actuator_ctrlrange[i][0]), m.actuator_ctrlrange[i][1])
        j = int(m.actuator_trnid[i])
        a, d = int(m.jnt_qposadr[j]), int(m.jnt_dofadr[j])
        gear = float(np.ravel(m.actuator_gear[i])[0])
        f = m.actuator_gainprm[i][0] * c
        if m.actuator_biastype[i]:
            bp = m.actuator_biasprm[i]
            f += bp[0] + bp[1] * (q[a] * gear) + bp[2] * (qd[d] * gear)
        if m.actuator_forcelimited[i]:
            f = min(max(f, m.actuator_forcerange[i][0]), m.actuator_forcerange[i][1])
        force[i] = f
        qf[d] += gear * f
    return qf, force


class Forward:
    """every smooth-dynamics output of one state.  env: per-environment values {"body_mass": {b: v}, "body_inertia": {b: v3},
    "dof_damping": vec, "dof_armature": vec}; body_pose: {b: (pos, quat)} of world-welded bodies placed per environment"""

    def __init__(self, m, q, qd, ctrl=None, env=None, body_pose=None):
        env = env or {}
        q, qd = np.asarray(q, dtype=np.float64), np.asarray(qd, dtype=np.float64)
        ctrl = np.zeros(int(m.nu)) if ctrl is None else np.asarray(ctrl, dtype=np.float64)
        body = {b: (env.get("body_mass", {}).get(b, m.body_mass[b]), env.get("body_inertia", {}).get(b, m.body_inertia[b]))
                for b in set(env.get("body_mass", {})) | set(env.get("body_inertia", {}))}
        self.damping = np.asarray(env.get("dof_damping", m.dof_damping), dtype=np.float64)
        self.armature = np.asarray(env.get("dof_armature", m.dof_armature), dtype=np.float64)
        self.m, self.q, self.qd, self.ctrl = m, q, qd, ctrl
        self.kin = k = Kin(m, q, body_pose)
        self.xpos, self.xmat, self.xipos = k.xpos, k.xmat, k.xipos
        self.xquat = np.array([mat2quat(R) for R in k.xmat])
        self.geom_xpos = np.array([T[:3, 3] for T in k.geom]).reshape(-1, 3)
        self.geom_xmat = np.array([T[:3, :3] for T in k.geom]).reshape(-1, 3, 3)
        self.site_xpos = np.array([T[:3, 3] for T in k.site]).reshape(-1, 3)
        self.site_xmat = np.array([T[:3, :3] for T in k.site]).reshape(-1, 3, 3)
        self.cdof = k.cdof()
        self.M = mass_matrix(m, k, self.armature, body)
        self.qfrc_bias = rnea(m, k, qd, np.zeros(int(m.nv)), m.opt_gravity, body)
        self.qfrc_passive, self.qfrc_spring_damper, self.qfrc_fluid = passive(m, k, q, qd, self.damping, body)
        self.qfrc_actuator, self.actuator_force = actuation(m, q, qd, ctrl)
        self.qfrc_smooth = self.qfrc_passive - self.qfrc_bias + self.qfrc_actuator
        self.qacc_smooth = np.linalg.solve(self.M, self.qfrc_smooth)

    def euler(self, qfrc_constraint=None):
        """(qpos, qvel) after one semi-implicit Euler step"""
        m = self.m
        h = float(m.opt_timestep)
        rhs = self.qfrc_smooth + (0 if qfrc_constraint is None else qfrc_constraint)
        acc = np.linalg.solve(self.M + h * np.diag(self.damping), rhs)
        return integrate(m, self.q, self.qd + h * acc, h)


def integrate(m, q, qd_new, h):
    q = q.copy()
    for j in range(int(m.njnt)):
        a, d = int(m.jnt_qposadr[j]), int(m.jnt_dofadr[j])
        if int(m.jnt_type[j]) == FREE:
            q[a:a + 3] += h * qd_new[d:d + 3]
            r = qmul(q[a + 3:a + 7], qexp(qd_new[d + 3:d + 6], h))
            q[a + 3:a + 7] = r / np.linalg.norm(r)
        else:
            q[a] += h * qd_new[d]
    return q, qd_new
