"""Scenes, poses and exact fp64 references for the narrow-phase tests (test_cpu_narrow_phase.py, test_gpu_narrow_phase.py, and the
warm-start tests test_cpu_narrow_phase_warm.py and test_gpu_narrow_phase_warm.py).

A scene is one geom pair: a plane plus one free body, or two free bodies with one geom each.  The references are functions of the
geoms' world poses (as the kinematics place them) and sizes only, so they check the collision routines and nothing else:
- closed-form signed distances for plane-{sphere, capsule, ellipsoid, cylinder, box, mesh}, sphere-{sphere, box, capsule, cylinder}
  and capsule-capsule (segment-segment closest points from the interior stationary point and the four clamped end projections);
- box-box: the 15-axis separating-axis depth, which is the exact penetration depth of two boxes;
- every other pair: the minimum over unit directions u of the support function of the Minkowski difference,
  h_A(u) + h_B(-u).  Positive, it is the penetration depth; negative, minus the distance.  Brute force over a dense direction set,
  then a Nelder-Mead refinement from the best directions.  Any direction gives an upper bound, so the result can only be
  above the true value, by the refinement's tolerance.
Signed distances are negative when the geoms overlap, as a contact's `dist` is.
"""
import os
import tempfile

import numpy as np

TYPES = {"plane": 0, "sphere": 2, "capsule": 3, "ellipsoid": 4, "cylinder": 5, "box": 6, "mesh": 7}
SOLIDS = ["sphere", "capsule", "ellipsoid", "cylinder", "box", "mesh"]
SIZES = {"sphere": (0.03,), "capsule": (0.02, 0.06), "ellipsoid": (0.05, 0.03, 0.02), "cylinder": (0.03, 0.05),
         "box": (0.05, 0.04, 0.02)}
ANALYTIC = {("plane", t) for t in SOLIDS} | {("sphere", t) for t in ("sphere", "box", "capsule", "cylinder")} | {("capsule", "capsule"),
                                                                                                            ("box", "box")}
# most contacts one pair can produce (plane-box, plane-cylinder and plane-mesh: 4, box-box: 8, plane-capsule: one per end)
MAXCON = {("plane", "box"): 4, ("plane", "cylinder"): 4, ("plane", "mesh"): 4, ("box", "box"): 8, ("plane", "capsule"): 2}
# an irregular convex polyhedron (all points on its hull), metres; the compiler recentres it at its volume centroid
_MESH = np.array([[0.04, 0.0, 0.0], [-0.035, 0.0, 0.0], [0.0, 0.03, 0.0], [0.0, -0.028, 0.0], [0.0, 0.0, 0.025], [0.0, 0.0, -0.03],
                  [0.02, 0.018, 0.015], [-0.02, -0.016, 0.014], [0.022, -0.015, -0.018], [-0.018, 0.02, -0.016]])


def pair_types():
    """every geom type pair the compiler puts in the pair list, in collision order (lower type first)"""
    out = [("plane", t) for t in SOLIDS]
    for i, a in enumerate(SOLIDS):
        for b in SOLIDS[i:]:
            out.append((a, b))
    return out


def pair_name(pair):
    return "%s-%s" % pair


def _fib(n):
    i = np.arange(n) + 0.5
    phi = np.arccos(1 - 2 * i / n)
    th = np.pi * (1 + 5 ** 0.5) * i
    return np.stack([np.cos(th) * np.sin(phi), np.sin(th) * np.sin(phi), np.cos(phi)], axis=1)


def ellipsoid_hull(n, axes, seed, mirror=False):
    """n points on the ellipsoid with semi-axes `axes` (metres), at jittered Fibonacci directions: every point lies on a strictly
    convex surface, so every point is a hull vertex.  mirror: the second half is the first mirrored in y (equal support values
    for directions with no y component: argmax ties between vertices in different lanes of a warp)"""
    rng = np.random.default_rng(seed)
    m = n // 2 if mirror else n
    u = _fib(m) + rng.normal(scale=0.3 / np.sqrt(m), size=(m, 3))
    if mirror:
        u[:, 1] = np.maximum(np.abs(u[:, 1]), 0.05)  # strictly one side of y = 0: the mirror images are distinct points
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    p = u / np.sqrt(((u / np.asarray(axes)) ** 2).sum(axis=1, keepdims=True))
    if mirror:
        p = np.concatenate([p, p * [1.0, -1.0, 1.0]])
    return p


# the convex hulls of the narrow-phase scenes, by mesh name: the 10-vertex probe, and ellipsoidal hulls sized for the mesh support
# scan (32 lanes: several vertices per lane, ties across lanes) and for the convex kernel's hull staging (see staging_case)
HULLS = {"probe": _MESH,
         "hull200": ellipsoid_hull(200, (0.05, 0.035, 0.03), seed=1, mirror=True),
         "hull2000a": ellipsoid_hull(2000, (0.06, 0.04, 0.03), seed=2),
         "hull2000b": ellipsoid_hull(2000, (0.035, 0.05, 0.04), seed=3),
         "hull3000": ellipsoid_hull(3000, (0.07, 0.05, 0.035), seed=4)}

_MESH_DIR = []


def _write_obj(path, V):
    from scipy.spatial import ConvexHull

    hull = ConvexHull(V)
    faces = []
    for a, b, c in hull.simplices:  # counter-clockwise seen from outside: the mass properties need outward normals
        n = np.cross(V[b] - V[a], V[c] - V[a])
        faces.append((a, b, c) if n @ (V[a] - V.mean(axis=0)) > 0 else (a, c, b))
    with open(path, "w") as f:
        f.writelines("v %.17g %.17g %.17g\n" % tuple(v) for v in V)
        f.writelines("f %d %d %d\n" % tuple(np.array(t) + 1) for t in faces)


def _mesh_dir():
    """a private temporary directory holding every hull of HULLS as an OBJ file <name>.obj (removed at exit)"""
    if not _MESH_DIR:
        import atexit
        import shutil

        d = tempfile.mkdtemp(prefix="b2s_narrow_phase_")
        atexit.register(shutil.rmtree, d, True)
        for name, V in HULLS.items():
            _write_obj(os.path.join(d, name + ".obj"), V)
        _MESH_DIR.append(d)
    return _MESH_DIR[0]


def _geom_xml(t, size=None, extra="", mesh="probe"):
    if t == "mesh":
        return '<geom type="mesh" mesh="%s"%s/>' % (mesh, extra)
    sz = " ".join("%.17g" % s for s in (size or SIZES[t]))
    return '<geom type="%s" size="%s"%s/>' % (t, sz, extra)


def scene_xml(pair, sizes=(None, None), meshes=("probe", "probe"), far=None):
    """MJCF of one pair: geom 0 is the first type (a world plane, or on free body a), geom 1 the second (on free body b); a mesh
    geom k uses the hull HULLS[meshes[k]].  far: a third free body far away with the hull HULLS[far], in no pair (collision bits
    disjoint from the pair's), which only enlarges the model's hulls"""
    t1, t2 = pair
    used = sorted({meshes[k] for k in range(2) if pair[k] == "mesh"} | ({far} if far else set()))
    asset = '<asset>%s</asset>' % "".join('<mesh name="%s" file="%s.obj"/>' % (m, m) for m in used) if used else ""
    if t1 == "plane":
        bodies = ('<geom type="plane" size="1 1 0.1"/><body name="b" pos="0 0 0.5"><freejoint/>%s</body>'
                  % _geom_xml(t2, sizes[1], mesh=meshes[1]))
    else:
        bodies = ('<body name="a" pos="0 0 1"><freejoint/>%s</body><body name="b" pos="0 0 2"><freejoint/>%s</body>'
                  % (_geom_xml(t1, sizes[0], mesh=meshes[0]), _geom_xml(t2, sizes[1], mesh=meshes[1])))
    if far:
        bodies += '<body name="far" pos="0 0 5"><freejoint/>%s</body>' % _geom_xml("mesh", extra=' contype="2" conaffinity="2"', mesh=far)
    return '<mujoco><option timestep="0.002" cone="elliptic"/>%s<worldbody>%s</worldbody></mujoco>' % (asset, bodies)


# mesh-mesh scenes of the hulls above: name -> (meshes of geoms 0 and 1, the far body's hull or None).  Their staging cases per
# schedule and precision are HULL_STAGING (test_cpu_narrow_phase_warm.py derives them from the capacity formulas)
HULL_SCENES = {"probe-hull200": (("probe", "hull200"), None), "hull2000a-hull2000b": (("hull2000a", "hull2000b"), None),
               "hull3000-hull200": (("hull3000", "hull200"), None), "hull3000-hull3000": (("hull3000", "hull3000"), None),
               "probe-probe": (("probe", "probe"), None), "probe-probe+far200": (("probe", "probe"), "hull200"),
               "hull200-hull200": (("hull200", "hull200"), None)}
# the phase pipeline's staging case per scene: (f32, f64)
HULL_STAGING = {"probe-hull200": ("both", "both"), "hull2000a-hull2000b": ("both", "only A"),
                "hull3000-hull200": ("both", "only B"), "hull3000-hull3000": ("only A", "neither"),
                "probe-probe": ("only A", "only A"), "probe-probe+far200": ("same hull", "same hull"),
                "hull200-hull200": ("only A", "only A")}


def hull_poses(meshes, n, seed, tail=()):
    """(qpos [m, nq], ambiguous flags, names) of a mesh-mesh hull scene: n random poses around contact and a catalogue (coincident
    centres; unrotated hulls 2 mm into each other along x and deep along z: support directions without a y component, where the
    mirrored 200-vertex hull has ties); `tail`: the far body's qpos appended to each"""
    C = np.array([0, 0, 1.0])
    Q = list(random_poses(("mesh", "mesh"), n, seed, meshes=meshes))
    amb, names = [False] * n, ["random%d" % i for i in range(n)]
    A, B = HULLS[meshes[0]], HULLS[meshes[1]]
    gx = A[:, 0].max() - B[:, 0].min() - 0.002
    gz = 0.6 * (A[:, 2].max() - B[:, 2].min())
    for name, q, a in [("concentric", _two(C, I4, C, I4), True), ("concentric_rotated", _two(C, axq([1, 2, 3], 0.7), C, axq([3, -1, 2], 1.1)), True),
                       ("x_2mm", _two(C, I4, C + [gx, 0, 0], I4), False), ("z_deep", _two(C, I4, C + [0.003, 0, gz], I4), False),
                       ("deep_offset", _two(C, axq([1, 0, 0], 0.3), C + [0.006, -0.004, 0.008], axq([0, 1, 1], 0.5)), False)]:
        Q.append(q); amb.append(a); names.append(name)
    return np.array([np.concatenate([q, tail]) for q in Q]), amb, names


def compile_scene(xml):
    from robosuite_b200.mjcf.compiler import compile_mjcf

    return compile_mjcf(xml, mesh_root=_mesh_dir() if "<mesh " in xml else None)


# ------------------------------------------------------------------------------------------------ hull staging
# The convex narrow phase of the phase pipeline (mode 1) and of the unit queue (mode 2) copies a pair's two poses (24 reals) and, where
# they fit, its hulls into shared memory before GJK (convex_convex in b2s_collide.cuh).  The pipeline's area holds the model's two
# largest hulls, at most 56 KB (b2s_capi.cu); the unit queue's is what its per-warp workspace leaves beside the EPA polytope
# (b2s_unit.cuh), used from 64 reals on.
EPA_AREA_WORDS = (9 * 96 + 5 * 192 + 64 + 8 + 40 + 3) & ~3
STAGING_CASES = ("both", "only A", "only B", "neither", "same hull")


def _pad4(k):
    return (k + 3) & ~3


def pipeline_stage_cap(vertnums, prec):
    """the phase pipeline's staging capacity in reals from the model's mesh_vertnum"""
    n = sorted(vertnums, reverse=True) + [0, 0]
    return min(24 + _pad4(3 * n[0]) + _pad4(3 * n[1]), 56 * 1024 // (8 if prec == "f64" else 4))


def unit_stage_cap(stride_words):
    """the unit queue's staging capacity in reals from its per-warp workspace stride (0: no staging)"""
    cap = stride_words - EPA_AREA_WORDS
    return cap if cap >= 64 else 0


def staging_case(nA, nB, same, cap):
    """which hulls convex_convex stages for hulls of nA and nB vertices (same: two instances of one mesh) in `cap` reals"""
    if cap <= 0:
        return "neither"
    cap -= 24
    a = 3 * nA <= cap
    used = _pad4(3 * nA) if a else 0
    b = used + 3 * nB <= cap
    if a and b:
        return "same hull" if same else "both"
    return "only A" if a else ("only B" if b else "neither")


# ------------------------------------------------------------------------------------------------ rotations
def quat2mat(q):
    w, x, y, z = np.asarray(q, dtype=np.float64) / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def axq(axis, ang):
    axis = np.asarray(axis, dtype=np.float64)
    axis = axis / np.linalg.norm(axis)
    return np.concatenate([[np.cos(ang / 2)], np.sin(ang / 2) * axis])


I4 = np.array([1.0, 0, 0, 0])


# ------------------------------------------------------------------------------------------------ geoms
class Geom:
    """one geom in the world: type name, size (3), world position, world rotation (columns = local axes), hull vertices (mesh)"""

    def __init__(self, t, size, pos, mat, vert=None):
        self.t, self.size, self.pos, self.mat, self.vert = t, np.asarray(size, dtype=np.float64), np.asarray(pos, dtype=np.float64), \
            np.asarray(mat, dtype=np.float64).reshape(3, 3), vert

    def extent(self, D):
        """support function about the centre, for unit directions D [n, 3]"""
        D = np.atleast_2d(D)
        L = D @ self.mat
        s = self.size
        if self.t == "sphere":
            return np.full(len(D), s[0])
        if self.t == "capsule":
            return s[1] * np.abs(L[:, 2]) + s[0]
        if self.t == "ellipsoid":
            return np.linalg.norm(L * s, axis=1)
        if self.t == "cylinder":
            return s[1] * np.abs(L[:, 2]) + s[0] * np.sqrt(np.maximum(L[:, 0] ** 2 + L[:, 1] ** 2, 0))
        if self.t == "box":
            return (np.abs(L) * s).sum(axis=1)
        if self.t == "mesh":  # in blocks of directions: [n, nvert] at once is gigabytes for the large hulls
            return np.concatenate([(L[k:k + 2048] @ self.vert.T).max(axis=1) for k in range(0, len(L), 2048)])
        if self.t == "point":
            return np.zeros(len(D))
        if self.t == "segment":
            return s[1] * np.abs(L[:, 2])
        raise ValueError(self.t)

    def support(self, D):
        D = np.atleast_2d(D)
        return self.extent(D) + D @ self.pos

    @property
    def radius(self):
        """the radius the narrow phase inflates the core by: spheres and capsules; 0 otherwise"""
        return float(self.size[0]) if self.t in ("sphere", "capsule") else 0.0

    def core(self):
        """the shape GJK runs on: a sphere's centre point, a capsule's segment, every other geom itself"""
        if self.t == "sphere":
            return Geom("point", self.size, self.pos, self.mat)
        if self.t == "capsule":
            return Geom("segment", self.size, self.pos, self.mat)
        return self


def separation_along(A, B, v):
    """min over a in A of u.a minus max over b in B of u.b, u = v / |v|: positive when the direction separates A from B (a GJK
    direction v points from B towards A: it is a point of the Minkowski difference A - B)"""
    u = np.asarray(v, dtype=np.float64) / np.linalg.norm(v)
    return float(-A.support(-u[None])[0] - B.support(u[None])[0])


def core_distance(A, B):
    """signed distance of the two cores (negative: they overlap by that depth); closed forms for points and segments"""
    ca, cb = A.core(), B.core()
    if ca.t in ("point", "segment") and cb.t in ("point", "segment"):
        ha = ca.size[1] if ca.t == "segment" else 0.0
        hb = cb.size[1] if cb.t == "segment" else 0.0
        return seg_seg_dist(ca.pos, ca.mat[:, 2], ha, cb.pos, cb.mat[:, 2], hb)
    return -mink_depth(ca, cb)


def geoms_of(model, o):
    """the scene's geoms at the oracle's current kinematics (o.forward() done)"""
    out = []
    inv = {v: k for k, v in TYPES.items()}
    for g in range(model.ngeom):
        t = inv[int(model.geom_type[g])]
        vert = None
        if t == "mesh":
            m = int(model.geom_dataid[g])
            a, n = int(model.mesh_vertadr[m]), int(model.mesh_vertnum[m])
            vert = np.array(model.mesh_vert[a:a + n], dtype=np.float64)
        out.append(Geom(t, model.geom_size[g], o.geom_xpos[g].copy(), o.geom_xmat[g].reshape(3, 3).copy(), vert))
    return out


# ------------------------------------------------------------------------------------------------ exact signed distances
_DIRS = _fib(20000)


def support_min(f, extra_dirs=()):
    """min over unit u of f(u) (f takes [n, 3]): brute force over 20,000 directions, then Nelder-Mead on the tangent plane of the
    two best directions and of `extra_dirs` (candidate directions only tighten the upper bound)"""
    from scipy.optimize import minimize

    v = f(_DIRS)
    starts = list(_DIRS[np.argsort(v)[:2]]) + [np.asarray(d, dtype=np.float64) / np.linalg.norm(d) for d in extra_dirs]
    best = float(v.min())
    for d0 in starts:
        e1 = np.cross(d0, [1.0, 0, 0] if abs(d0[0]) < 0.6 else [0, 1.0, 0])
        e1 /= np.linalg.norm(e1)
        e2 = np.cross(d0, e1)

        def g(x):
            u = d0 + x[0] * e1 + x[1] * e2
            return float(f(u[None] / np.linalg.norm(u))[0])

        r = minimize(g, np.zeros(2), method="Nelder-Mead",
                     options=dict(xatol=1e-12, fatol=1e-15, maxiter=2000, initial_simplex=[[0, 0], [0.03, 0], [0, 0.03]]))
        best = min(best, float(r.fun), g(np.zeros(2)))
    return best


def mink_depth(A, B, extra_dirs=()):
    """min_u h_A(u) + h_B(-u): the penetration depth (> 0) or minus the distance (< 0)"""
    return support_min(lambda D: A.support(D) + B.support(-D), extra_dirs)


def _seg_point(a, u, h, p):
    return a + u * np.clip((p - a) @ u, -h, h)


def seg_seg_dist(a, u, ha, b, v, hb):
    """distance of the segments a + s u (|s| <= ha), b + t v (|t| <= hb): least of the interior stationary point and the four
    projections of one segment's ends onto the other (the minimum of a convex quadratic on a box lies on one of these)"""
    cands = []
    for s in (-ha, ha):
        p = a + s * u
        cands.append(np.linalg.norm(p - _seg_point(b, v, hb, p)))
    for t in (-hb, hb):
        q = b + t * v
        cands.append(np.linalg.norm(q - _seg_point(a, u, ha, q)))
    M = np.array([[u @ u, -u @ v], [-u @ v, v @ v]])
    if abs(np.linalg.det(M)) > 1e-14:
        s, t = np.linalg.solve(M, [-(a - b) @ u, (a - b) @ v])
        if abs(s) <= ha and abs(t) <= hb:
            cands.append(np.linalg.norm(a + s * u - b - t * v))
    return min(cands)


def point_sd(G, p):
    """signed distance of the point p to the solid G (negative inside)"""
    if G.t == "plane":
        return (p - G.pos) @ G.mat[:, 2]
    l = G.mat.T @ (p - G.pos)
    s = G.size
    if G.t == "sphere":
        return np.linalg.norm(l) - s[0]
    if G.t == "capsule":
        return np.linalg.norm(l - np.array([0, 0, np.clip(l[2], -s[1], s[1])])) - s[0]
    if G.t == "box":
        q = np.abs(l) - s[:3]
        return np.linalg.norm(np.maximum(q, 0)) + min(q.max(), 0)
    if G.t == "cylinder":
        q = np.array([np.hypot(l[0], l[1]) - s[0], abs(l[2]) - s[1]])
        return np.linalg.norm(np.maximum(q, 0)) + min(q.max(), 0)
    return -support_min(lambda D: G.support(D) - D @ p)  # ellipsoid, mesh


def sat_depth(A, B):
    """box-box: least overlap over the 15 separating axes (> 0 overlapping: the penetration depth; <= 0 separated)"""
    axes = [A.mat[:, i] for i in range(3)] + [B.mat[:, i] for i in range(3)]
    for i in range(3):
        for j in range(3):
            x = np.cross(A.mat[:, i], B.mat[:, j])
            if np.linalg.norm(x) > 1e-9:
                axes.append(x / np.linalg.norm(x))
    return min(min(float(A.support(L)[0] + B.support(-L)[0]), float(A.support(-L)[0] + B.support(L)[0])) for L in axes)


def signed_distance(A, B, extra_dirs=()):
    """exact signed distance of the pair (negative: penetration depth).  Box-box separated: the largest axis separation (a lower
    bound of the distance with the right sign)."""
    if A.t == "plane":
        n = A.mat[:, 2]
        return float((B.pos - A.pos) @ n - B.extent(-n[None])[0])
    if (A.t, B.t) == ("box", "box"):
        return -sat_depth(A, B)
    if A.t == "sphere" and B.t in ("sphere", "box", "capsule", "cylinder"):
        return float(point_sd(B, A.pos) - A.size[0])
    if (A.t, B.t) == ("capsule", "capsule"):
        return seg_seg_dist(A.pos, A.mat[:, 2], A.size[1], B.pos, B.mat[:, 2], B.size[1]) - A.size[0] - B.size[0]
    return -mink_depth(A, B, extra_dirs)


def overlap_along(A, B, n):
    """overlap of the pair's projections on n: shifting B by this much along n separates them along n"""
    n = np.asarray(n, dtype=np.float64)[None]
    if A.t == "plane":
        return float(-((B.pos - A.pos) @ n[0]) + B.extent(-n)[0])
    return float(A.support(n)[0] + B.support(-n)[0])


# ------------------------------------------------------------------------------------------------ poses
def _rand_quat(rng):
    q = rng.normal(size=4)
    return q / np.linalg.norm(q)


def _rbound(t, size, mesh="probe"):
    if t == "mesh":
        return float(np.linalg.norm(HULLS[mesh], axis=1).max())
    s = np.asarray(size or SIZES[t], dtype=np.float64)
    return {"sphere": s[0], "capsule": s[0] + s[-1], "ellipsoid": s.max(), "cylinder": np.hypot(s[0], s[-1]),
            "box": np.linalg.norm(s)}[t]


def random_poses(pair, n, seed, sizes=(None, None), meshes=("probe", "probe")):
    """n seeded qpos around contact: geom 2's centre at a random direction from geom 1 (or above the plane), at a distance between
    deep overlap and a little beyond touching"""
    rng = np.random.default_rng(seed)
    t1, t2 = pair
    out = []
    for _ in range(n):
        qb = _rand_quat(rng)
        if t1 == "plane":
            if t2 == "mesh":
                ext = _rbound(t2, None, meshes[1])
            else:
                ext = float(Geom(t2, _pad(sizes[1] or SIZES[t2]), np.zeros(3), quat2mat(qb)).extent(np.array([[0, 0, -1.0]]))[0])
            z = ext * rng.uniform(0.4, 1.15)
            out.append(np.concatenate([[rng.uniform(-0.2, 0.2), rng.uniform(-0.2, 0.2), z], qb]))
        else:
            qa = _rand_quat(rng)
            d = rng.normal(size=3)
            d /= np.linalg.norm(d)
            r = (_rbound(t1, sizes[0], meshes[0]) + _rbound(t2, sizes[1], meshes[1])) * rng.uniform(0.15, 0.9)
            pa = np.array([0, 0, 1.0])
            out.append(np.concatenate([pa, qa, pa + r * d, qb]))
    return np.array(out)


def _pad(s):
    s = list(s)
    return s + [0.0] * (3 - len(s))


def _two(pa, qa, pb, qb):
    return np.concatenate([pa, qa, pb, qb])


def catalogue(pair):
    """named degenerate configurations of a pair: [(name, qpos, ambiguous)].  An ambiguous contact (coincident centres, intersecting
    cores, two equally good reference faces) has no unique normal or position: only the depth and the contact invariants hold it, not a
    comparison of normals and positions between implementations."""
    t1, t2 = pair
    C = np.array([0, 0, 1.0])
    out = []
    r45 = axq([0, 0, 1], np.pi / 4)
    if t1 == "plane":
        s = SIZES.get(t2)
        if t2 == "capsule":
            out += [("horizontal_1mm", np.concatenate([[0, 0, s[0] - 0.001], axq([0, 1, 0], np.pi / 2)]), False),
                    ("upright_1mm", np.concatenate([[0, 0, s[0] + s[1] - 0.001], I4]), False),
                    ("tilted_deep", np.concatenate([[0, 0, 0.02], axq([1, 0, 0], 0.4)]), False)]
        if t2 == "ellipsoid":
            out += [("flat_1mm", np.concatenate([[0, 0, s[2] - 0.001], I4]), False),
                    ("tilted_1mm", np.concatenate([[0, 0, 0.0], axq([1, 1, 0], 0.7)]), False)]
        if t2 == "cylinder":
            out += [("upright_1mm", np.concatenate([[0, 0, s[1] - 0.001], I4]), False),
                    ("lying_1mm", np.concatenate([[0, 0, s[0] - 0.001], axq([1, 0, 0], np.pi / 2)]), False),
                    ("tilted_1mm", np.concatenate([[0, 0, s[1] * np.cos(0.5) + s[0] * np.sin(0.5) - 0.001], axq([1, 0, 0], 0.5)]), False),
                    ("upright_deep", np.concatenate([[0, 0, 0.2 * s[1]], I4]), False)]
        if t2 == "box":
            out += [("face_1mm", np.concatenate([[0, 0, s[2] - 0.001], I4]), False),
                    ("vertex_1mm", np.concatenate([[0, 0, np.linalg.norm(s) - 0.001],
                                                   axq(np.cross(s, [0, 0, 1.0]), np.arccos(s[2] / np.linalg.norm(s)))]), False),
                    ("edge_45", np.concatenate([[0, 0, np.hypot(s[1], s[2]) - 0.002], axq([1, 0, 0], np.arctan2(s[1], s[2]))]), False),
                    ("face_deep", np.concatenate([[0, 0, 0.3 * s[2]], I4]), False)]
        if t2 == "sphere":
            out += [("touch", np.concatenate([[0, 0, s[0]], I4]), False), ("deep", np.concatenate([[0, 0, 0.2 * s[0]], I4]), False)]
        if t2 == "mesh":
            out += [("deep", np.concatenate([[0, 0, 0.005], I4]), False), ("tilted", np.concatenate([[0, 0, 0.02], axq([1, 2, 0], 0.9)]), False)]
        return out
    # coincident centres: every pair at its deepest; the normal is only ambiguous where both shapes are symmetric about it
    out.append(("concentric", _two(C, I4, C, I4), True))
    out.append(("concentric_rotated", _two(C, axq([1, 2, 3], 0.7), C, axq([3, -1, 2], 1.1)), True))
    if pair == ("sphere", "sphere"):
        out += [("touch", _two(C, I4, C + [0.05, 0, 0], I4), False), ("offset_1mm", _two(C, I4, C + [0, 0, 0.049], I4), False)]
    if pair == ("sphere", "box"):
        out += [("inside_off_centre", _two(C + [0.01, 0.005, 0.002], I4, C, axq([0, 0, 1], 0.3)), False),
                ("face_touch", _two(C + [0, 0, 0.05], I4, C, I4), False),
                ("vertex_region", _two(C + [0.06, 0.05, 0.03], I4, C, I4), False)]
    if pair == ("sphere", "cylinder"):
        out += [("on_axis_near_cap", _two(C + [0, 0, 0.04], I4, C, I4), False),
                ("on_axis_beyond_cap", _two(C + [0, 0, 0.07], I4, C, I4), False),
                ("rim", _two(C + [0.04, 0, 0.06], I4, C, I4), False)]
    if pair == ("sphere", "capsule"):
        for off in (0.045, 0.03, 0.01):
            out.append(("axis_offset_%g" % off, _two(C + [off, 0, 0.02], I4, C, I4), False))
        out += [("on_segment", _two(C + [0, 0, 0.03], I4, C, I4), True),
                ("beyond_end", _two(C + [0, 0, 0.1], I4, C, I4), False)]
    if pair == ("capsule", "capsule"):
        cross = axq([0, 1, 0], np.pi / 2)  # a along x, b along z
        for off in (0.035, 0.005):
            out.append(("crossing_offset_%g" % off, _two(C, cross, C + [0, off, 0], I4), False))
        out += [("crossing_axes_meet", _two(C, cross, C, I4), True),
                ("crossing_axes_meet_off_centre", _two(C, cross, C + [0.03, 0, 0.02], I4), True),
                ("collinear_overlap", _two(C, I4, C + [0, 0, 0.05], I4), True),
                ("parallel_offset", _two(C, I4, C + [0.03, 0, 0.05], I4), False),
                ("end_to_end_1mm", _two(C, I4, C + [0, 0, 0.159], I4), False),
                ("skew", _two(C, axq([1, 0, 0], 0.3), C + [0.01, 0.02, 0.01], axq([0, 1, 0], 1.2)), False)]
    if pair == ("box", "box"):
        sa, sb = np.array(SIZES["box"]), np.array(SIZES["box"])
        out += [("stacked_aligned_1mm", _two(C, I4, C + [0, 0, sa[2] + sb[2] - 0.001], I4), False),
                ("stacked_offset_1mm", _two(C, I4, C + [0.03, -0.02, sa[2] + sb[2] - 0.001], I4), False),
                ("stacked_rotated_45", _two(C, I4, C + [0, 0, sa[2] + sb[2] - 0.002], r45), False),
                ("side_by_side", _two(C, I4, C + [2 * sa[0] - 0.003, 0.01, 0.0], I4), True)]  # either box's face is the reference
        qa, qb = axq([1, 0, 0], np.pi / 4), axq([0, 1, 0], np.pi / 4)
        ha = (sa[1] + sa[2]) / np.sqrt(2)  # half-heights after the 45 degree turns: a's top edge along x, b's bottom edge along y
        hb = (sb[0] + sb[2]) / np.sqrt(2)
        out.append(("edge_edge_45", _two(C, qa, C + [0, 0, ha + hb - 0.002], qb), False))
        v = sb / np.linalg.norm(sb)
        qv = axq(np.cross(v, [0, 0, -1.0]), np.arccos(-v[2]))  # vertex (+,+,+) of b pointing down
        out.append(("vertex_on_face", _two(C, I4, C + [0.01, 0.01, sa[2] + np.linalg.norm(sb) - 0.002], qv), False))
    if t2 in ("cylinder", "box", "mesh", "ellipsoid", "capsule") and pair not in (("capsule", "capsule"), ("sphere", "capsule")):
        out.append(("deep_offset", _two(C, axq([1, 0, 0], 0.3), C + [0.006, -0.004, 0.008], axq([0, 1, 1], 0.5)), False))
    if pair == ("cylinder", "cylinder"):
        out += [("stacked_1mm", _two(C, I4, C + [0, 0, 0.099], I4), False), ("side_1mm", _two(C, I4, C + [0.059, 0, 0], I4), False),
                ("crossed", _two(C, axq([1, 0, 0], np.pi / 2), C + [0, 0, 0.055], axq([0, 1, 0], np.pi / 2)), False)]
    if pair == ("box", "cylinder"):
        out += [("cylinder_upright_on_box", _two(C, I4, C + [0.01, 0, 0.069], I4), False),
                ("cylinder_lying_on_box", _two(C, I4, C + [0, 0.01, 0.049], axq([1, 0, 0], np.pi / 2)), False)]
    return out


def size_variants(pair, scales=(0.7, 1.3)):
    """per-environment sizes: each primitive's size scaled to the ends of a +-30 % randomisation range"""
    out = []
    for k in scales:
        sz = tuple(None if t in ("plane", "mesh") else tuple(k * np.array(SIZES[t])) for t in pair)
        out.append((k, sz))
    return out


# ------------------------------------------------------------------------------------------------ checks
def check_contacts(pair, A, B, cons, ref, tol):
    """invariants of one pair's contacts against the exact signed distance `ref`; returns a list of failures.
    cons: [(dist, pos[3], frame[3x3])]; tol: dict(band, depth, pos, frame, sep, rel): depth, pos and sep gates are
    tol[...] + tol["rel"] * |ref| (tol["sep_rel"] for sep)"""
    bad = []
    tol = dict(tol)
    for k in ("depth", "pos", "sep"):
        tol[k] += tol.get("sep_rel" if k == "sep" else "rel", 0.0) * abs(ref)
    lim = MAXCON.get(pair, 1)
    if len(cons) > lim:
        bad.append("%d contacts > %d" % (len(cons), lim))
    if ref < -tol["band"] and not cons:
        bad.append("missing contact at exact dist %.3g" % ref)
    if ref > tol["band"] and cons:
        bad.append("contact at exact dist %.3g" % ref)
    if not cons:
        return bad
    for dist, pos, fr in cons:
        fr = np.asarray(fr, dtype=np.float64).reshape(3, 3)
        if dist > 0:
            bad.append("dist %.3g > 0" % dist)
        e = np.abs(fr @ fr.T - np.eye(3)).max()
        if e > tol["frame"] or np.linalg.det(fr) < 0:
            bad.append("frame not orthonormal (%.3g)" % e)
        pos = np.asarray(pos, dtype=np.float64)
        for G in (A, B):
            if pair == ("plane", "capsule"):  # each contact belongs to one end sphere of the capsule
                ends = [B.pos + k * B.size[1] * B.mat[:, 2] for k in (1, -1)]
                G = G if G is A else Geom("sphere", B.size, min(ends, key=lambda e: np.linalg.norm(e - pos)), B.mat)
            d = abs(point_sd(G, pos))
            if d > abs(dist) / 2 + tol["pos"]:
                bad.append("pos %.3g from the %s surface, |dist|/2 = %.3g" % (d, G.t, abs(dist) / 2))
    deepest = min(cons, key=lambda c: c[0])
    dmin, n = deepest[0], np.asarray(deepest[2], dtype=np.float64).reshape(3, 3)[0]
    ov = overlap_along(A, B, n)
    if pair == ("box", "box"):
        sat = -ref
        if not (sat - tol["depth"] <= -dmin <= 1.05 * sat + 1e-5 + tol["depth"]):
            bad.append("box-box depth %.9g outside [SAT %.9g, 1.05 SAT + 1e-5]" % (-dmin, sat))
        # the face-clipped manifold can miss the reference face's deepest incident vertex: its normal is then checked against the
        # face-preference bound rather than against the deepest contact
        if ov > 1.05 * sat + 1e-5 + tol["sep"]:
            bad.append("normal's axis overlap %.9g beyond 1.05 SAT + 1e-5 (SAT %.9g)" % (ov, sat))
    elif abs(dmin - ref) > tol["depth"]:
        bad.append("deepest dist %.12g vs exact %.12g (err %.3g)" % (dmin, ref, abs(dmin - ref)))
    if pair != ("box", "box") and ov > -dmin + tol["sep"]:
        bad.append("normal does not separate: overlap along n %.9g > -dist %.9g" % (ov, -dmin))
    return bad
