"""MJCF -> flat model arrays (host side, compile time).

Replaces the reference's call into the third-party engine's XML compiler
(`robosuite/utils/binding_utils.py:1079` `mujoco.MjModel.from_xml_string`, reached from
`robosuite/environments/base.py:255-275`).  Input is the *composed* MJCF the reference's Python model layer emits
(`robosuite/models/base.py:83-158`); the feature universe handled is exactly the one those documents use
(SURVEY.md section 8 a-0).  Field names follow the `mjModel` attribute names the reference reads through
`binding_utils.MjModel` so the same arrays back the MjSim-compatible facade.

Id ordering: bodies / joints / geoms / sites are numbered in depth-first document order, world body = 0, which is
what the reference's name<->id maps (`binding_utils.py:326-360`) observe from the engine.
"""
import math
import os
import xml.etree.ElementTree as ET

import numpy as np

from . import meshio

# object / joint / geom type enums (values match the engine enums the reference compares against,
# e.g. `binding_utils.py:511-534` uses mjtJoint.mjJNT_FREE etc.)
JNT_FREE, JNT_BALL, JNT_SLIDE, JNT_HINGE = 0, 1, 2, 3
GEOM_PLANE, GEOM_HFIELD, GEOM_SPHERE, GEOM_CAPSULE, GEOM_ELLIPSOID, GEOM_CYLINDER, GEOM_BOX, GEOM_MESH = range(8)
GEOM_TYPES = {"plane": 0, "hfield": 1, "sphere": 2, "capsule": 3, "ellipsoid": 4, "cylinder": 5, "box": 6, "mesh": 7}
MINVAL = 1e-15


# ----------------------------------------------------------------------------------------------- small math
def _vec(s, n=None, default=None):
    if s is None:
        return None if default is None else np.array(default, dtype=np.float64)
    v = np.array([float(t) for t in s.split()], dtype=np.float64)
    if n is not None and len(v) != n:
        if default is not None and len(v) < n:
            d = np.array(default, dtype=np.float64)
            d[: len(v)] = v
            return d
        raise ValueError(f"expected {n} values, got '{s}'")
    return v


def quat_mul(a, b):
    return np.array([
        a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3],
        a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
        a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1],
        a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0],
    ])


def quat2mat(q):
    w, x, y, z = q
    return np.array([
        [w * w + x * x - y * y - z * z, 2 * (x * y - w * z), 2 * (x * z + w * y)],
        [2 * (x * y + w * z), w * w - x * x + y * y - z * z, 2 * (y * z - w * x)],
        [2 * (x * z - w * y), 2 * (y * z + w * x), w * w - x * x - y * y + z * z],
    ])


def mat2quat(R):
    # robust conversion (w,x,y,z), w >= 0 branch selection by largest diagonal
    t = np.trace(R)
    if t > 0:
        s = math.sqrt(t + 1.0) * 2
        q = np.array([0.25 * s, (R[2, 1] - R[1, 2]) / s, (R[0, 2] - R[2, 0]) / s, (R[1, 0] - R[0, 1]) / s])
    elif R[0, 0] > R[1, 1] and R[0, 0] > R[2, 2]:
        s = math.sqrt(1.0 + R[0, 0] - R[1, 1] - R[2, 2]) * 2
        q = np.array([(R[2, 1] - R[1, 2]) / s, 0.25 * s, (R[0, 1] + R[1, 0]) / s, (R[0, 2] + R[2, 0]) / s])
    elif R[1, 1] > R[2, 2]:
        s = math.sqrt(1.0 + R[1, 1] - R[0, 0] - R[2, 2]) * 2
        q = np.array([(R[0, 2] - R[2, 0]) / s, (R[0, 1] + R[1, 0]) / s, 0.25 * s, (R[1, 2] + R[2, 1]) / s])
    else:
        s = math.sqrt(1.0 + R[2, 2] - R[0, 0] - R[1, 1]) * 2
        q = np.array([(R[1, 0] - R[0, 1]) / s, (R[0, 2] + R[2, 0]) / s, (R[1, 2] + R[2, 1]) / s, 0.25 * s])
    return q / np.linalg.norm(q)


def axisangle2quat(axis, angle):
    n = np.linalg.norm(axis)
    if n < MINVAL:
        return np.array([1.0, 0, 0, 0])
    a = axis / n
    return np.concatenate([[math.cos(angle / 2)], a * math.sin(angle / 2)])


def z2quat(vec):
    """quaternion rotating (0,0,1) onto vec"""
    v = vec / np.linalg.norm(vec)
    axis = np.cross([0.0, 0.0, 1.0], v)
    s = np.linalg.norm(axis)
    if s < 1e-10:
        return np.array([1.0, 0, 0, 0]) if v[2] > 0 else np.array([0.0, 1.0, 0, 0])
    ang = math.atan2(s, v[2])
    return axisangle2quat(axis / s, ang)


def _orientation(el, use_degree=False, eulerseq="xyz"):
    q = el.get("quat")
    if q is not None:
        q = _vec(q, 4)
        return q / np.linalg.norm(q)
    aa = el.get("axisangle")
    if aa is not None:
        aa = _vec(aa, 4)
        ang = math.radians(aa[3]) if use_degree else aa[3]
        return axisangle2quat(aa[:3], ang)
    eu = el.get("euler")
    if eu is not None:
        eu = _vec(eu, 3)
        if use_degree:
            eu = np.radians(eu)
        q = np.array([1.0, 0, 0, 0])
        for ch, a in zip(eulerseq, eu):
            ax = {"x": [1, 0, 0], "y": [0, 1, 0], "z": [0, 0, 1]}[ch.lower()]
            r = axisangle2quat(np.array(ax, dtype=float), a)
            q = quat_mul(q, r) if ch.islower() else quat_mul(r, q)
        return q / np.linalg.norm(q)
    xy = el.get("xyaxes")
    if xy is not None:
        xy = _vec(xy, 6)
        x = xy[:3] / np.linalg.norm(xy[:3])
        y = xy[3:] - x * np.dot(x, xy[3:])
        y /= np.linalg.norm(y)
        return mat2quat(np.stack([x, y, np.cross(x, y)], axis=1))
    za = el.get("zaxis")
    if za is not None:
        return z2quat(_vec(za, 3))
    return np.array([1.0, 0, 0, 0])


def eig3_desc(I):
    """Principal axes of a symmetric 3x3: eigenvalues sorted descending + right-handed rotation quaternion."""
    w, V = np.linalg.eigh(I)
    order = np.argsort(-w, kind="stable")
    w, V = w[order], V[:, order]
    if np.linalg.det(V) < 0:
        V[:, 2] = -V[:, 2]
    return w, mat2quat(V)


# ----------------------------------------------------------------------------------------------- model container
class Model:
    """Flat compiled model.  Attributes are numpy arrays / scalars named like the engine's mjModel fields."""

    def __init__(self):
        self.names = {}  # objtype -> list of names (None for unnamed)

    def arrays(self):
        return {k: v for k, v in self.__dict__.items() if isinstance(v, np.ndarray)}

    def scalars(self):
        return {k: v for k, v in self.__dict__.items() if isinstance(v, (int, float)) and not isinstance(v, bool)}

    def name2id(self, objtype, name):
        try:
            return self.names[objtype].index(name)
        except ValueError:
            return -1


# ----------------------------------------------------------------------------------------------- compile
def primitive_geom_props(t, sz):
    """(volume, inertia diagonal per unit mass in the geom frame, bounding radius, local box [centre 3, half sizes 3]) of a primitive
    geom of type t and size sz.  The set-constants pass (b2s_set_const) applies the same bound rules to per-environment sizes."""
    vol, I, rbound, aabb = 0.0, np.zeros(3), 0.0, [0, 0, 0, 0, 0, 0]
    if t == GEOM_SPHERE:
        r = sz[0]
        vol = 4.0 / 3.0 * math.pi * r ** 3
        I[:] = 0.4 * r * r
        rbound = r
        aabb = [0, 0, 0, r, r, r]
    elif t == GEOM_BOX:
        vol = 8 * sz[0] * sz[1] * sz[2]
        I = np.array([sz[1] ** 2 + sz[2] ** 2, sz[0] ** 2 + sz[2] ** 2, sz[0] ** 2 + sz[1] ** 2]) / 3.0
        rbound = np.linalg.norm(sz)
        aabb = [0, 0, 0, sz[0], sz[1], sz[2]]
    elif t == GEOM_CYLINDER:
        r, h = sz[0], sz[1]
        vol = math.pi * r * r * 2 * h
        I = np.array([(3 * r * r + 4 * h * h) / 12.0, (3 * r * r + 4 * h * h) / 12.0, r * r / 2.0])
        rbound = math.sqrt(r * r + h * h)
        aabb = [0, 0, 0, r, r, h]
    elif t == GEOM_CAPSULE:
        r, h = sz[0], sz[1]
        vc = math.pi * r * r * 2 * h
        vs = 4.0 / 3.0 * math.pi * r ** 3
        vol = vc + vs
        izz = (vc * r * r / 2 + vs * 0.4 * r * r) / vol
        ixx = (vc * (3 * r * r + 4 * h * h) / 12 + vs * (0.4 * r * r + h * h + 0.75 * r * h)) / vol
        I = np.array([ixx, ixx, izz])
        rbound = r + h
        aabb = [0, 0, 0, r, r, r + h]
    elif t == GEOM_ELLIPSOID:
        vol = 4.0 / 3.0 * math.pi * sz[0] * sz[1] * sz[2]
        I = np.array([sz[1] ** 2 + sz[2] ** 2, sz[0] ** 2 + sz[2] ** 2, sz[0] ** 2 + sz[1] ** 2]) / 5.0
        rbound = sz.max()
        aabb = [0, 0, 0, sz[0], sz[1], sz[2]]
    elif t == GEOM_PLANE:
        rbound = 0.0
        aabb = [0, 0, -1e10, 1e10, 1e10, 1e10]
    return vol, I, rbound, aabb


def compile_mjcf(xml_string: str, mesh_root: str = None) -> Model:
    from ..errors import XMLError

    try:
        root = ET.fromstring(xml_string)
    except ET.ParseError as e:  # the reference surfaces the engine's XML errors to the caller (SURVEY section 8b)
        raise XMLError("MJCF parse error: %s" % e) from e
    if root.tag != "mujoco":
        raise XMLError("root element is <%s>, expected <mujoco>" % root.tag)
    comp = root.find("compiler")
    comp = comp.attrib if comp is not None else {}
    use_degree = comp.get("angle", "degree") == "degree"
    eulerseq = comp.get("eulerseq", "xyz")
    autolimits = comp.get("autolimits", "true") == "true"
    igr = _vec(comp.get("inertiagrouprange"), 2, [0, 5]).astype(int)
    meshdir = comp.get("meshdir", "")
    opt = root.find("option")
    opt = opt.attrib if opt is not None else {}

    m = Model()
    m.opt_timestep = float(opt.get("timestep", 0.002))
    m.opt_impratio = float(opt.get("impratio", 1.0))
    m.opt_density = float(opt.get("density", 0.0))
    m.opt_viscosity = float(opt.get("viscosity", 0.0))
    m.opt_tolerance = float(opt.get("tolerance", 1e-8))
    m.opt_iterations = int(opt.get("iterations", 100))
    m.opt_ls_iterations = int(opt.get("ls_iterations", 50))
    m.opt_ls_tolerance = float(opt.get("ls_tolerance", 0.01))
    m.opt_cone = 1 if opt.get("cone", "pyramidal") == "elliptic" else 0
    m.opt_gravity = _vec(opt.get("gravity"), 3, [0, 0, -9.81])
    m.opt_wind = _vec(opt.get("wind"), 3, [0, 0, 0])
    if opt.get("integrator", "Euler") != "Euler":
        raise NotImplementedError("only the Euler integrator is implemented")
    if opt.get("solver", "Newton") != "Newton":
        raise NotImplementedError("only the Newton solver is implemented")

    # ---------------- assets: meshes
    mesh_names, mesh_data = [], []
    asset = root.find("asset")
    if asset is not None:
        for me in asset.findall("mesh"):
            fn = me.get("file")
            if not os.path.isabs(fn):
                fn = os.path.join(mesh_root or "", meshdir, fn)
            name = me.get("name") or os.path.splitext(os.path.basename(fn))[0]
            mesh_names.append(name)
            mesh_data.append(dict(file=fn, scale=_vec(me.get("scale"), 3, [1, 1, 1]), loaded=None))

    def get_mesh(mid):
        md = mesh_data[mid]
        if md["loaded"] is None:
            v, f = meshio.load_mesh(md["file"])
            v = v * md["scale"][None, :]
            if np.prod(md["scale"]) < 0:
                f = f[:, ::-1]
            try:
                hv, hf = meshio.convex_hull(v)
            except Exception:  # degenerate (flat) visual meshes: keep the raw vertices
                hv, hf = v, f
            md["loaded"] = dict(vert=v, face=f, hull_vert=hv, hull_face=hf)
        return md["loaded"]

    # ---------------- bodies (DFS)
    B = dict(name=[], parent=[], pos=[], quat=[], mocap=[], inertial=[], el=[])
    J = []  # joints
    G = []  # geoms
    S = []  # sites
    CAM, LIGHT = [], []

    def add_body(el, parent):
        bid = len(B["name"])
        B["name"].append(el.get("name") if bid else "world")
        B["parent"].append(parent)
        B["pos"].append(_vec(el.get("pos"), 3, [0, 0, 0]) if bid else np.zeros(3))
        B["quat"].append(_orientation(el, use_degree, eulerseq) if bid else np.array([1.0, 0, 0, 0]))
        B["mocap"].append(el.get("mocap", "false") == "true")
        B["inertial"].append(el.find("inertial"))
        if float(el.get("gravcomp", 0)) != 0:
            raise NotImplementedError("body gravcomp is not implemented")
        for ch in el:
            if ch.tag in ("joint", "freejoint"):
                J.append((bid, ch))
            elif ch.tag == "geom":
                G.append((bid, ch))
            elif ch.tag == "site":
                S.append((bid, ch))
            elif ch.tag == "camera":
                CAM.append((bid, ch))
            elif ch.tag == "light":
                LIGHT.append((bid, ch))
        for ch in el:
            if ch.tag == "body":
                add_body(ch, bid)

    # the engine lists a body's own elements before recursing; joints/geoms/sites therefore come out in DFS order
    # but grouped per body -> collect per body first, then flatten in body order
    add_body(root.find("worldbody"), 0)
    nbody = len(B["name"])
    J.sort(key=lambda t: t[0])
    G.sort(key=lambda t: t[0])
    S.sort(key=lambda t: t[0])
    CAM.sort(key=lambda t: t[0])
    LIGHT.sort(key=lambda t: t[0])

    m.nbody = nbody
    m.body_parentid = np.array(B["parent"], dtype=np.int32)
    m.body_pos = np.array(B["pos"])
    m.body_quat = np.array(B["quat"])
    m.names["body"] = B["name"]
    mocapid = -np.ones(nbody, dtype=np.int32)
    k = 0
    for i in range(nbody):
        if B["mocap"][i]:
            mocapid[i] = k
            k += 1
    m.body_mocapid = mocapid
    m.nmocap = k

    # ---------------- joints / dofs
    njnt = len(J)
    jnt_type = np.zeros(njnt, dtype=np.int32)
    jnt_bodyid = np.zeros(njnt, dtype=np.int32)
    jnt_qposadr = np.zeros(njnt, dtype=np.int32)
    jnt_dofadr = np.zeros(njnt, dtype=np.int32)
    jnt_pos = np.zeros((njnt, 3))
    jnt_axis = np.zeros((njnt, 3))
    jnt_axis[:, 2] = 1
    jnt_range = np.zeros((njnt, 2))
    jnt_limited = np.zeros(njnt, dtype=np.int32)
    jnt_margin = np.zeros(njnt)
    jnt_stiffness = np.zeros(njnt)
    jnt_solref = np.tile([0.02, 1.0], (njnt, 1))
    jnt_solimp = np.tile([0.9, 0.95, 0.001, 0.5, 2.0], (njnt, 1))
    dof = dict(body=[], jnt=[], armature=[], damping=[], frictionloss=[], solref=[], solimp=[])
    qpos0 = []
    qpos_spring = []  # spring reference: springref for hinge and slide joints, qpos0 for free and ball joints
    jnames = []
    nq = nv = 0
    for j, (bid, el) in enumerate(J):
        jnames.append(el.get("name"))
        t = "free" if el.tag == "freejoint" else el.get("type", "hinge")
        jt = {"free": JNT_FREE, "ball": JNT_BALL, "slide": JNT_SLIDE, "hinge": JNT_HINGE}[t]
        jnt_type[j] = jt
        jnt_bodyid[j] = bid
        jnt_qposadr[j] = nq
        jnt_dofadr[j] = nv
        jnt_pos[j] = _vec(el.get("pos"), 3, [0, 0, 0])
        ax = _vec(el.get("axis"), 3, [0, 0, 1])
        jnt_axis[j] = ax / max(np.linalg.norm(ax), MINVAL)
        rng = el.get("range")
        if rng is not None:
            r = _vec(rng, 2)
            if use_degree and jt == JNT_HINGE:
                r = np.radians(r)
            jnt_range[j] = r
        lim = el.get("limited", "auto")
        jnt_limited[j] = 1 if lim == "true" else 0 if lim == "false" else int(autolimits and rng is not None)
        jnt_margin[j] = float(el.get("margin", 0))
        jnt_stiffness[j] = float(el.get("stiffness", 0))
        if jt == JNT_FREE and jnt_stiffness[j] != 0:
            raise NotImplementedError("stiffness on a free joint is not implemented")
        if el.get("springdamper") is not None and np.any(_vec(el.get("springdamper"), 2) != 0):
            raise NotImplementedError("joint springdamper is not implemented")
        if el.get("solreflimit"):
            jnt_solref[j] = _vec(el.get("solreflimit"), 2)
        if el.get("solimplimit"):
            jnt_solimp[j] = _vec(el.get("solimplimit"), 5, [0.9, 0.95, 0.001, 0.5, 2.0])
        nd = {JNT_FREE: 6, JNT_BALL: 3, JNT_SLIDE: 1, JNT_HINGE: 1}[jt]
        nqj = {JNT_FREE: 7, JNT_BALL: 4, JNT_SLIDE: 1, JNT_HINGE: 1}[jt]
        if jt == JNT_FREE:
            # free joint: only allowed on children of world; qpos0 = body frame
            qpos0 += list(B["pos"][bid]) + list(B["quat"][bid])
            qpos_spring += qpos0[-7:]
            jnt_pos[j] = 0
        elif jt == JNT_BALL:
            qpos0 += [1.0, 0, 0, 0]
            qpos_spring += [1.0, 0, 0, 0]
        else:
            deg = math.pi / 180 if use_degree and jt == JNT_HINGE else 1.0  # a hinge's ref and springref are angles
            qpos0.append(float(el.get("ref", 0)) * deg)
            qpos_spring.append(float(el.get("springref", 0)) * deg)
        for _ in range(nd):
            dof["body"].append(bid)
            dof["jnt"].append(j)
            dof["armature"].append(float(el.get("armature", 0)))
            dof["damping"].append(float(el.get("damping", 0)))
            dof["frictionloss"].append(float(el.get("frictionloss", 0)))
            dof["solref"].append(_vec(el.get("solreffriction"), 2, [0.02, 1.0]))
            dof["solimp"].append(_vec(el.get("solimpfriction"), 5, [0.9, 0.95, 0.001, 0.5, 2.0]))
        nq += nqj
        nv += nd
    m.njnt, m.nq, m.nv = njnt, nq, nv
    m.jnt_type, m.jnt_bodyid, m.jnt_qposadr, m.jnt_dofadr = jnt_type, jnt_bodyid, jnt_qposadr, jnt_dofadr
    m.jnt_pos, m.jnt_axis, m.jnt_range, m.jnt_limited = jnt_pos, jnt_axis, jnt_range, jnt_limited
    m.jnt_margin, m.jnt_stiffness, m.jnt_solref, m.jnt_solimp = jnt_margin, jnt_stiffness, jnt_solref, jnt_solimp
    m.names["joint"] = jnames
    m.qpos0 = np.array(qpos0, dtype=np.float64)
    m.qpos_spring = np.array(qpos_spring, dtype=np.float64)
    m.dof_bodyid = np.array(dof["body"], dtype=np.int32)
    m.dof_jntid = np.array(dof["jnt"], dtype=np.int32)
    m.dof_armature = np.array(dof["armature"], dtype=np.float64)
    m.dof_damping = np.array(dof["damping"], dtype=np.float64)
    m.dof_frictionloss = np.array(dof["frictionloss"], dtype=np.float64)
    m.dof_solref = np.array(dof["solref"], dtype=np.float64).reshape(nv, 2)
    m.dof_solimp = np.array(dof["solimp"], dtype=np.float64).reshape(nv, 5)

    body_jntnum = np.zeros(nbody, dtype=np.int32)
    body_jntadr = -np.ones(nbody, dtype=np.int32)
    body_dofnum = np.zeros(nbody, dtype=np.int32)
    body_dofadr = -np.ones(nbody, dtype=np.int32)
    for j in range(njnt):
        b = jnt_bodyid[j]
        if body_jntnum[b] == 0:
            body_jntadr[b] = j
            body_dofadr[b] = jnt_dofadr[j]
        body_jntnum[b] += 1
    for d in range(nv):
        body_dofnum[m.dof_bodyid[d]] += 1
    m.body_jntnum, m.body_jntadr, m.body_dofnum, m.body_dofadr = body_jntnum, body_jntadr, body_dofnum, body_dofadr

    # kinematic-tree bookkeeping
    weld = np.zeros(nbody, dtype=np.int32)
    rootid = np.zeros(nbody, dtype=np.int32)
    for i in range(1, nbody):
        p = m.body_parentid[i]
        weld[i] = i if body_jntnum[i] > 0 else weld[p]
        rootid[i] = i if p == 0 else rootid[p]
    m.body_weldid, m.body_rootid = weld, rootid
    dof_parent = -np.ones(nv, dtype=np.int32)
    last_dof_of_body = -np.ones(nbody, dtype=np.int32)  # last dof on the chain ending at this body
    for i in range(1, nbody):
        last = last_dof_of_body[m.body_parentid[i]]
        for d in range(body_dofadr[i], body_dofadr[i] + body_dofnum[i]) if body_dofnum[i] else []:
            dof_parent[d] = last
            last = d
        last_dof_of_body[i] = last
    m.dof_parentid = dof_parent
    # sparse-M addressing: row i holds (i,i), (i,parent), (i,grandparent) ...
    madr = np.zeros(nv, dtype=np.int32)
    nM = 0
    for i in range(nv):
        madr[i] = nM
        d = i
        while d >= 0:
            nM += 1
            d = dof_parent[d]
    m.dof_Madr, m.nM = madr, nM

    # ---------------- geoms
    ngeom = len(G)
    g = dict(type=np.zeros(ngeom, dtype=np.int32), bodyid=np.zeros(ngeom, dtype=np.int32),
             contype=np.ones(ngeom, dtype=np.int32), conaffinity=np.ones(ngeom, dtype=np.int32),
             condim=3 * np.ones(ngeom, dtype=np.int32), group=np.zeros(ngeom, dtype=np.int32),
             priority=np.zeros(ngeom, dtype=np.int32), dataid=-np.ones(ngeom, dtype=np.int32),
             size=np.zeros((ngeom, 3)), pos=np.zeros((ngeom, 3)), quat=np.zeros((ngeom, 4)),
             friction=np.zeros((ngeom, 3)), solmix=np.ones(ngeom), solref=np.zeros((ngeom, 2)),
             solimp=np.zeros((ngeom, 5)), margin=np.zeros(ngeom), gap=np.zeros(ngeom), rbound=np.zeros(ngeom),
             aabb=np.zeros((ngeom, 6)), rgba=np.zeros((ngeom, 4)))
    gnames = []
    geom_mass = np.zeros(ngeom)
    geom_inertia_local = np.zeros((ngeom, 3, 3))  # inertia about geom COM, in geom frame axes
    geom_com_local = np.zeros((ngeom, 3))  # COM offset in geom frame (meshes only)
    for i, (bid, el) in enumerate(G):
        gnames.append(el.get("name"))
        t = GEOM_TYPES[el.get("type", "sphere")]
        g["type"][i] = t
        g["bodyid"][i] = bid
        g["contype"][i] = int(el.get("contype", 1))
        g["conaffinity"][i] = int(el.get("conaffinity", 1))
        g["condim"][i] = int(el.get("condim", 3))
        g["group"][i] = int(el.get("group", 0))
        g["priority"][i] = int(el.get("priority", 0))
        g["friction"][i] = _vec(el.get("friction"), 3, [1, 0.005, 0.0001])
        g["solmix"][i] = float(el.get("solmix", 1))
        g["solref"][i] = _vec(el.get("solref"), 2, [0.02, 1.0])
        g["solimp"][i] = _vec(el.get("solimp"), 5, [0.9, 0.95, 0.001, 0.5, 2.0])
        g["margin"][i] = float(el.get("margin", 0))
        g["gap"][i] = float(el.get("gap", 0))
        g["rgba"][i] = _vec(el.get("rgba"), 4, [0.5, 0.5, 0.5, 1])
        size = _vec(el.get("size"), None, None)
        sz = np.zeros(3)
        if size is not None:
            sz[: len(size)] = size
        pos = _vec(el.get("pos"), 3, [0, 0, 0])
        quat = _orientation(el, use_degree, eulerseq)
        ft = el.get("fromto")
        if ft is not None:
            ft = _vec(ft, 6)
            vec = ft[:3] - ft[3:]
            pos = 0.5 * (ft[:3] + ft[3:])
            quat = z2quat(vec)
            half = 0.5 * np.linalg.norm(vec)
            if t in (GEOM_CAPSULE, GEOM_CYLINDER):
                sz[1] = half
            else:
                sz[2] = half
        g["size"][i], g["pos"][i], g["quat"][i] = sz, pos, quat
        density = float(el.get("density", 1000))
        if t == GEOM_MESH:
            vol, I = 0.0, np.zeros(3)
            mid = mesh_names.index(el.get("mesh"))
            g["dataid"][i] = mid
        else:
            vol, I, g["rbound"][i], g["aabb"][i] = primitive_geom_props(t, sz)
        Il = np.diag(I)
        if t == GEOM_MESH:
            md = get_mesh(g["dataid"][i])
            hv = md["hull_vert"]
            g["rbound"][i] = np.linalg.norm(hv, axis=1).max()
            lo, hi = hv.min(axis=0), hv.max(axis=0)
            g["aabb"][i] = np.concatenate([(lo + hi) / 2, (hi - lo) / 2])
            vol, com, Im = meshio.mesh_mass_properties(md["vert"], md["face"])
            geom_com_local[i] = com
            Il = Im / vol if vol > 0 else np.zeros((3, 3))
        if el.get("mass") is not None:
            geom_mass[i] = float(el.get("mass"))
        else:
            geom_mass[i] = density * vol
        geom_inertia_local[i] = Il * geom_mass[i]
    m.ngeom = ngeom
    for k_, v_ in g.items():
        setattr(m, "geom_" + k_, v_)
    m.names["geom"] = gnames
    body_geomnum = np.zeros(nbody, dtype=np.int32)
    body_geomadr = -np.ones(nbody, dtype=np.int32)
    for i in range(ngeom):
        b = g["bodyid"][i]
        if body_geomnum[b] == 0:
            body_geomadr[b] = i
        body_geomnum[b] += 1
    m.body_geomnum, m.body_geomadr = body_geomnum, body_geomadr

    # ---------------- meshes used for collision: pack hull vertices
    m.names["mesh"] = mesh_names
    nmesh = len(mesh_names)
    vertadr = np.zeros(nmesh, dtype=np.int32)
    vertnum = np.zeros(nmesh, dtype=np.int32)
    verts = []
    nvt = 0
    used = set(int(x) for x in g["dataid"] if x >= 0)
    # only meshes referenced by geoms that can collide are needed on the path
    coll = set(int(g["dataid"][i]) for i in range(ngeom)
               if g["dataid"][i] >= 0 and (g["contype"][i] or g["conaffinity"][i]))
    for mid in range(nmesh):
        vertadr[mid] = nvt
        if mid in coll:
            hv = get_mesh(mid)["hull_vert"]
            verts.append(hv)
            vertnum[mid] = len(hv)
            nvt += len(hv)
    m.nmesh = nmesh
    m.mesh_vertadr, m.mesh_vertnum = vertadr, vertnum
    m.mesh_vert = np.concatenate(verts, axis=0) if verts else np.zeros((0, 3))
    m.nmeshvert = nvt

    # ---------------- body inertial properties
    body_mass = np.zeros(nbody)
    body_ipos = np.zeros((nbody, 3))
    body_iquat = np.tile([1.0, 0, 0, 0], (nbody, 1))
    body_inertia = np.zeros((nbody, 3))
    for b in range(1, nbody):
        iel = B["inertial"][b]
        if iel is not None:
            body_mass[b] = float(iel.get("mass"))
            body_ipos[b] = _vec(iel.get("pos"), 3, [0, 0, 0])
            if iel.get("fullinertia") is not None:
                fi = _vec(iel.get("fullinertia"), 6)
                Ifull = np.array([[fi[0], fi[3], fi[4]], [fi[3], fi[1], fi[5]], [fi[4], fi[5], fi[2]]])
                w, q = eig3_desc(Ifull)
                body_inertia[b] = w
                body_iquat[b] = quat_mul(_orientation(iel, use_degree, eulerseq), q)
            else:
                body_inertia[b] = _vec(iel.get("diaginertia"), 3, [0, 0, 0])
                body_iquat[b] = _orientation(iel, use_degree, eulerseq)
            continue
        idx = [i for i in range(ngeom) if g["bodyid"][i] == b and igr[0] <= g["group"][i] <= igr[1]
               and geom_mass[i] > 0]
        if not idx:
            continue
        mt = sum(geom_mass[i] for i in idx)
        coms = {}
        for i in idx:
            R = quat2mat(g["quat"][i])
            coms[i] = g["pos"][i] + R @ geom_com_local[i]
        com = sum(geom_mass[i] * coms[i] for i in idx) / mt
        Ib = np.zeros((3, 3))
        for i in idx:
            R = quat2mat(g["quat"][i])
            d = coms[i] - com
            Ib += R @ geom_inertia_local[i] @ R.T + geom_mass[i] * (np.dot(d, d) * np.eye(3) - np.outer(d, d))
        w, q = eig3_desc(Ib)
        body_mass[b], body_ipos[b], body_inertia[b], body_iquat[b] = mt, com, w, q
    m.body_mass, m.body_ipos, m.body_iquat, m.body_inertia = body_mass, body_ipos, body_iquat, body_inertia
    sub = body_mass.copy()
    for b in range(nbody - 1, 0, -1):
        sub[m.body_parentid[b]] += sub[b]
    m.body_subtreemass = sub

    # ---------------- sites
    nsite = len(S)
    m.nsite = nsite
    m.site_bodyid = np.array([b for b, _ in S], dtype=np.int32).reshape(nsite)
    m.site_pos = np.array([_vec(e.get("pos"), 3, [0, 0, 0]) for _, e in S]).reshape(nsite, 3)
    m.site_quat = np.array([_orientation(e, use_degree, eulerseq) for _, e in S]).reshape(nsite, 4)
    m.site_size = np.array([_vec(e.get("size"), 3, [0.005, 0.005, 0.005]) for _, e in S]).reshape(nsite, 3)
    m.site_rgba = np.array([_vec(e.get("rgba"), 4, [0.5, 0.5, 0.5, 1]) for _, e in S]).reshape(nsite, 4)
    m.names["site"] = [e.get("name") for _, e in S]
    m.names["camera"] = [e.get("name") for _, e in CAM]
    m.names["light"] = [e.get("name") for _, e in LIGHT]
    m.ncam, m.nlight = len(CAM), len(LIGHT)
    m.cam_bodyid = np.array([b for b, _ in CAM], dtype=np.int32).reshape(len(CAM))
    m.cam_pos = np.array([_vec(e.get("pos"), 3, [0, 0, 0]) for _, e in CAM]).reshape(len(CAM), 3)
    m.cam_quat = np.array([_orientation(e, use_degree, eulerseq) for _, e in CAM]).reshape(len(CAM), 4)
    m.cam_fovy = np.array([float(e.get("fovy", 45)) for _, e in CAM]).reshape(len(CAM))

    # ---------------- actuators
    A = []
    act = root.find("actuator")
    if act is not None:
        A = [e for e in act if e.tag in ("motor", "position", "velocity", "general")]
    nu = len(A)
    m.nu = nu
    m.actuator_trnid = np.zeros(nu, dtype=np.int32)
    m.actuator_ctrllimited = np.zeros(nu, dtype=np.int32)
    m.actuator_forcelimited = np.zeros(nu, dtype=np.int32)
    m.actuator_ctrlrange = np.zeros((nu, 2))
    m.actuator_forcerange = np.zeros((nu, 2))
    m.actuator_gear = np.zeros((nu, 6))
    m.actuator_gainprm = np.zeros((nu, 3))
    m.actuator_biasprm = np.zeros((nu, 3))
    m.actuator_biastype = np.zeros(nu, dtype=np.int32)  # 0 none, 1 affine
    anames = []
    for i, e in enumerate(A):
        anames.append(e.get("name"))
        jn = e.get("joint")
        for attr, ok in (("dyntype", ("none",)), ("gaintype", ("fixed",)), ("biastype", ("none", "affine"))):
            if e.get(attr, ok[0]) not in ok:
                raise NotImplementedError("actuator %s=%s is not implemented" % (attr, e.get(attr)))
        if jn is None:
            raise NotImplementedError("only joint transmissions are implemented")
        m.actuator_trnid[i] = jnames.index(jn)
        m.actuator_gear[i, 0] = _vec(e.get("gear"), None, None)[0] if e.get("gear") else 1.0
        cr, fr = e.get("ctrlrange"), e.get("forcerange")
        if cr:
            m.actuator_ctrlrange[i] = _vec(cr, 2)
        if fr:
            m.actuator_forcerange[i] = _vec(fr, 2)
        cl, fl = e.get("ctrllimited", "auto"), e.get("forcelimited", "auto")
        m.actuator_ctrllimited[i] = 1 if cl == "true" else 0 if cl == "false" else int(autolimits and cr is not None)
        m.actuator_forcelimited[i] = 1 if fl == "true" else 0 if fl == "false" else int(autolimits and fr is not None)
        if e.tag == "motor":
            m.actuator_gainprm[i, 0] = 1.0
        elif e.tag == "position":
            kp = float(e.get("kp", 1))
            kv = float(e.get("kv", 0))
            m.actuator_gainprm[i, 0] = kp
            m.actuator_biasprm[i] = [0, -kp, -kv]
            m.actuator_biastype[i] = 1
        elif e.tag == "velocity":
            kv = float(e.get("kv", 1))
            m.actuator_gainprm[i, 0] = kv
            m.actuator_biasprm[i] = [0, 0, -kv]
            m.actuator_biastype[i] = 1
        else:
            m.actuator_gainprm[i] = _vec(e.get("gainprm"), 3, [1, 0, 0])
            m.actuator_biasprm[i] = _vec(e.get("biasprm"), 3, [0, 0, 0])
            m.actuator_biastype[i] = 1 if e.get("biastype", "none") == "affine" else 0
    m.names["actuator"] = anames

    # ---------------- sensors (force / torque only; values are produced by the engine's post-constraint pass)
    SN = []
    sen = root.find("sensor")
    if sen is not None:
        SN = [e for e in sen if e.tag in ("force", "torque")]
    m.nsensor = len(SN)
    m.sensor_type = np.array([0 if e.tag == "force" else 1 for e in SN], dtype=np.int32).reshape(len(SN))
    m.sensor_objid = np.array([m.names["site"].index(e.get("site")) for e in SN], dtype=np.int32).reshape(len(SN))
    m.sensor_dim = 3 * np.ones(len(SN), dtype=np.int32)
    m.sensor_adr = 3 * np.arange(len(SN), dtype=np.int32)
    m.nsensordata = 3 * len(SN)
    m.names["sensor"] = [e.get("name") for e in SN]

    # ---------------- static collision pair list (contype/conaffinity, same weld body, welded parent-child)
    pairs = []
    for a in range(ngeom):
        for b in range(a + 1, ngeom):
            if not ((g["contype"][a] & g["conaffinity"][b]) or (g["contype"][b] & g["conaffinity"][a])):
                continue
            b1, b2 = g["bodyid"][a], g["bodyid"][b]
            w1, w2 = weld[b1], weld[b2]
            if w1 == w2:
                continue
            p1, p2 = weld[m.body_parentid[w1]], weld[m.body_parentid[w2]]
            if w1 != 0 and w2 != 0 and (w1 == p2 or w2 == p1):
                continue
            if g["type"][a] == GEOM_PLANE and g["type"][b] == GEOM_PLANE:
                continue
            pairs.append((a, b))
    m.pair_geom = np.array(pairs, dtype=np.int32).reshape(-1, 2)
    m.npair = len(pairs)

    _set_const(m)
    return m


# ----------------------------------------------------------------------------------------------- qpos0 constants
def _kin0(m, qpos):
    """Forward kinematics at qpos (numpy, compile-time helper): world pose of bodies, inertial frames, joint
    anchors/axes."""
    nb = m.nbody
    xpos = np.zeros((nb, 3))
    xquat = np.tile([1.0, 0, 0, 0], (nb, 1))
    xanchor = np.zeros((m.njnt, 3))
    xaxis = np.zeros((m.njnt, 3))
    for b in range(1, nb):
        p = m.body_parentid[b]
        Rp = quat2mat(xquat[p])
        pos = xpos[p] + Rp @ m.body_pos[b]
        quat = quat_mul(xquat[p], m.body_quat[b])
        for j in range(m.body_jntadr[b], m.body_jntadr[b] + m.body_jntnum[b]) if m.body_jntnum[b] else []:
            qa = m.jnt_qposadr[j]
            t = m.jnt_type[j]
            if t == JNT_FREE:
                pos = qpos[qa:qa + 3].copy()
                quat = qpos[qa + 3:qa + 7] / np.linalg.norm(qpos[qa + 3:qa + 7])
                xanchor[j] = pos
                xaxis[j] = [0, 0, 1]
                continue
            R = quat2mat(quat)
            xanchor[j] = pos + R @ m.jnt_pos[j]
            xaxis[j] = R @ m.jnt_axis[j]
            if t == JNT_SLIDE:
                pos = pos + xaxis[j] * (qpos[qa] - m.qpos0[qa])
            elif t == JNT_HINGE:
                quat = quat_mul(quat, axisangle2quat(m.jnt_axis[j], qpos[qa] - m.qpos0[qa]))
                pos = xanchor[j] - quat2mat(quat) @ m.jnt_pos[j]
            elif t == JNT_BALL:
                quat = quat_mul(quat, qpos[qa:qa + 4] / np.linalg.norm(qpos[qa:qa + 4]))
                pos = xanchor[j] - quat2mat(quat) @ m.jnt_pos[j]
        xpos[b], xquat[b] = pos, quat / np.linalg.norm(quat)
    return xpos, xquat, xanchor, xaxis


def _dof_axes(m, xpos, xquat, xanchor, xaxis):
    """Per-dof (angular axis, point on axis or None for translation) in world frame."""
    out = []
    for d in range(m.nv):
        j = m.dof_jntid[d]
        t = m.jnt_type[j]
        k = d - m.jnt_dofadr[j]
        b = m.jnt_bodyid[j]
        if t == JNT_FREE:
            if k < 3:
                e = np.zeros(3)
                e[k] = 1
                out.append((None, e, None))
            else:
                R = quat2mat(xquat[b])
                out.append((R[:, k - 3], None, xpos[b]))
        elif t == JNT_BALL:
            R = quat2mat(xquat[b])
            out.append((R[:, k], None, xanchor[j]))
        elif t == JNT_SLIDE:
            out.append((None, xaxis[j], None))
        else:
            out.append((xaxis[j], None, xanchor[j]))
    return out


def _jac_point(m, axes, body, point):
    """3 x nv translational and rotational Jacobians of a world point attached to `body`."""
    jp = np.zeros((3, m.nv))
    jr = np.zeros((3, m.nv))
    b = body
    while b > 0 and m.body_dofnum[b] == 0:
        b = m.body_parentid[b]
    if b == 0:
        return jp, jr
    d = m.body_dofadr[b] + m.body_dofnum[b] - 1
    while d >= 0:
        w, v, a = axes[d]
        if w is None:
            jp[:, d] = v
        else:
            jr[:, d] = w
            jp[:, d] = np.cross(w, point - a)
        d = m.dof_parentid[d]
    return jp, jr


def _mass_matrix(m, xpos, xquat, axes):
    """Dense joint-space inertia via sum_b J_b^T I_b J_b (compile-time helper; O(nbody nv^2))."""
    M = np.zeros((m.nv, m.nv))
    for b in range(1, m.nbody):
        if m.body_mass[b] <= 0 and not np.any(m.body_inertia[b] > 0):
            continue
        R = quat2mat(xquat[b])
        com = xpos[b] + R @ m.body_ipos[b]
        Ri = R @ quat2mat(m.body_iquat[b])
        Iw = Ri @ np.diag(m.body_inertia[b]) @ Ri.T
        jp, jr = _jac_point(m, axes, b, com)
        M += m.body_mass[b] * jp.T @ jp + jr.T @ Iw @ jr
    M += np.diag(m.dof_armature)
    return M


def _set_const(m):
    """Constants derived at qpos0 that the soft-constraint model needs: dof_invweight0, body_invweight0, dof_M0,
    actuator_acc0, stat_meaninertia (the engine computes these in its set-constants pass after compiling)."""
    nv = m.nv
    xpos, xquat, xanchor, xaxis = _kin0(m, m.qpos0)
    axes = _dof_axes(m, xpos, xquat, xanchor, xaxis)
    m.body_invweight0 = np.zeros((m.nbody, 2))
    m.dof_invweight0 = np.zeros(nv)
    m.dof_M0 = np.zeros(nv)
    m.actuator_acc0 = np.zeros(m.nu)
    m.stat_meaninertia = 1.0
    if nv == 0:
        return
    M = _mass_matrix(m, xpos, xquat, axes)
    Minv = np.linalg.inv(M)
    m.dof_M0 = np.diag(M).copy()
    m.stat_meaninertia = float(np.mean(np.diag(M)))
    diw = np.diag(Minv).copy()
    for j in range(m.njnt):
        a = m.jnt_dofadr[j]
        if m.jnt_type[j] == JNT_FREE:
            diw[a:a + 3] = diw[a:a + 3].mean()
            diw[a + 3:a + 6] = diw[a + 3:a + 6].mean()
        elif m.jnt_type[j] == JNT_BALL:
            diw[a:a + 3] = diw[a:a + 3].mean()
    m.dof_invweight0 = diw
    for b in range(1, m.nbody):
        if m.body_weldid[b] == 0:
            continue
        R = quat2mat(xquat[b])
        com = xpos[b] + R @ m.body_ipos[b]
        jp, jr = _jac_point(m, axes, b, com)
        Jb = np.vstack([jp, jr])
        A = Jb @ Minv @ Jb.T
        m.body_invweight0[b, 0] = (A[0, 0] + A[1, 1] + A[2, 2]) / 3
        m.body_invweight0[b, 1] = (A[3, 3] + A[4, 4] + A[5, 5]) / 3
    for i in range(m.nu):
        j = m.actuator_trnid[i]
        mom = np.zeros(nv)
        mom[m.jnt_dofadr[j]] = m.actuator_gear[i, 0]
        m.actuator_acc0[i] = np.linalg.norm(Minv @ mom)


# ----------------------------------------------------------------------------------------------- blob (de)serialise
_BLOB_MAGIC = b"B2SMODEL"


def pack_model(m: Model) -> bytes:
    """Serialise to the flat container both C sides read: magic, count, then records
    (name[48], dtype code i32 {0:f64,1:i32}, ndim i32, shape[4] i32, byte offset i64, nbytes i64), then 16B-aligned data.
    Scalars are stored as 1-element arrays."""
    import struct

    items = []
    for k, v in sorted(m.scalars().items()):
        a = np.array([v], dtype=np.int32 if isinstance(v, int) else np.float64)
        items.append((k, a))
    # name tables (MjModel name2id / id2name, binding_utils.py:362-492): per object type one '\n'-joined UTF-8 string as an i32 array of
    # byte values ("names_body", "names_joint", ...); unnamed objects are empty strings
    for objtype, lst in sorted(getattr(m, "names", {}).items()):
        joined = "\n".join("" if x is None else str(x) for x in lst).encode("utf-8")
        items.append(("names_" + objtype, np.frombuffer(joined, dtype=np.uint8).astype(np.int32) if joined else np.zeros(0, np.int32)))
    for k, v in sorted(m.arrays().items()):
        if v.dtype.kind in "iub":
            a = np.ascontiguousarray(v, dtype=np.int32)
        else:
            a = np.ascontiguousarray(v, dtype=np.float64)
        items.append((k, a))
    rec_size = 48 + 4 + 4 + 16 + 8 + 8
    head = 16 + rec_size * len(items)
    off = (head + 15) // 16 * 16
    recs, datas = [], []
    for k, a in items:
        shape = list(a.shape) + [0] * (4 - a.ndim)
        nb = a.nbytes
        recs.append(struct.pack("<48sii4iqq", k.encode()[:47], 0 if a.dtype == np.float64 else 1, a.ndim, *shape, off, nb))
        datas.append((off, a.tobytes()))
        off = (off + nb + 15) // 16 * 16
    buf = bytearray(off)
    buf[0:8] = _BLOB_MAGIC
    buf[8:16] = struct.pack("<q", len(items))
    p = 16
    for r in recs:
        buf[p:p + rec_size] = r
        p += rec_size
    for o, d in datas:
        buf[o:o + len(d)] = d
    return bytes(buf)


def save_model(m: Model, path: str):
    """Portable fixture: npz of arrays + scalars + names (the compiled model travels to boxes without mesh files)."""
    import json

    d = dict(m.arrays())
    d["__scalars__"] = np.frombuffer(json.dumps(m.scalars()).encode(), dtype=np.uint8)
    d["__names__"] = np.frombuffer(json.dumps(m.names).encode(), dtype=np.uint8)
    np.savez_compressed(path, **d)


def load_model(path: str) -> Model:
    import json

    z = np.load(path)
    m = Model()
    for k in z.files:
        if k == "__scalars__":
            for kk, vv in json.loads(bytes(z[k]).decode()).items():
                setattr(m, kk, vv)
        elif k == "__names__":
            m.names = json.loads(bytes(z[k]).decode())
        else:
            setattr(m, k, z[k])
    if not hasattr(m, "qpos_spring"):
        # written before the compiler recorded springref: those compilers sprang every joint back to qpos0, and the packaged
        # models (robosuite_b200/assets/models) have springref = ref = 0 on every joint
        m.qpos_spring = np.array(m.qpos0, dtype=np.float64)
    return m
