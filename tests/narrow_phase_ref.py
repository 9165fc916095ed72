"""Scenes, poses and exact fp64 references for the narrow-phase tests (test_cpu_narrow_phase.py, test_gpu_narrow_phase.py).

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


_MESH_DIR = []


def _mesh_dir():
    """a private temporary directory holding the probe mesh as an OBJ file (removed at exit)"""
    if not _MESH_DIR:
        import atexit
        import shutil

        from scipy.spatial import ConvexHull

        d = tempfile.mkdtemp(prefix="b2s_narrow_phase_")
        atexit.register(shutil.rmtree, d, True)
        hull = ConvexHull(_MESH)
        faces = []
        for a, b, c in hull.simplices:  # counter-clockwise seen from outside: the mass properties need outward normals
            n = np.cross(_MESH[b] - _MESH[a], _MESH[c] - _MESH[a])
            faces.append((a, b, c) if n @ (_MESH[a] - _MESH.mean(axis=0)) > 0 else (a, c, b))
        with open(os.path.join(d, "probe.obj"), "w") as f:
            f.writelines("v %.17g %.17g %.17g\n" % tuple(v) for v in _MESH)
            f.writelines("f %d %d %d\n" % tuple(np.array(t) + 1) for t in faces)
        _MESH_DIR.append(d)
    return _MESH_DIR[0]


def _geom_xml(t, size=None, extra=""):
    if t == "mesh":
        return '<geom type="mesh" mesh="probe"%s/>' % extra
    sz = " ".join("%.17g" % s for s in (size or SIZES[t]))
    return '<geom type="%s" size="%s"%s/>' % (t, sz, extra)


def scene_xml(pair, sizes=(None, None)):
    """MJCF of one pair: geom 0 is the first type (a world plane, or on free body a), geom 1 the second (on free body b)"""
    t1, t2 = pair
    asset = '<asset><mesh name="probe" file="probe.obj"/></asset>' if "mesh" in pair else ""
    if t1 == "plane":
        bodies = '<geom type="plane" size="1 1 0.1"/><body name="b" pos="0 0 0.5"><freejoint/>%s</body>' % _geom_xml(t2, sizes[1])
    else:
        bodies = ('<body name="a" pos="0 0 1"><freejoint/>%s</body><body name="b" pos="0 0 2"><freejoint/>%s</body>'
                  % (_geom_xml(t1, sizes[0]), _geom_xml(t2, sizes[1])))
    return '<mujoco><option timestep="0.002" cone="elliptic"/>%s<worldbody>%s</worldbody></mujoco>' % (asset, bodies)


def compile_scene(xml):
    from robosuite_b200.mjcf.compiler import compile_mjcf

    return compile_mjcf(xml, mesh_root=_mesh_dir() if 'mesh="probe"' in xml else None)


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
        if self.t == "mesh":
            return (L @ self.vert.T).max(axis=1)
        raise ValueError(self.t)

    def support(self, D):
        D = np.atleast_2d(D)
        return self.extent(D) + D @ self.pos


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
def _fib(n):
    i = np.arange(n) + 0.5
    phi = np.arccos(1 - 2 * i / n)
    th = np.pi * (1 + 5 ** 0.5) * i
    return np.stack([np.cos(th) * np.sin(phi), np.sin(th) * np.sin(phi), np.cos(phi)], axis=1)


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


def _rbound(t, size):
    if t == "mesh":
        return float(np.linalg.norm(_MESH, axis=1).max())
    s = np.asarray(size or SIZES[t], dtype=np.float64)
    return {"sphere": s[0], "capsule": s[0] + s[-1], "ellipsoid": s.max(), "cylinder": np.hypot(s[0], s[-1]),
            "box": np.linalg.norm(s)}[t]


def random_poses(pair, n, seed, sizes=(None, None)):
    """n seeded qpos around contact: geom 2's centre at a random direction from geom 1 (or above the plane), at a distance between
    deep overlap and a little beyond touching"""
    rng = np.random.default_rng(seed)
    t1, t2 = pair
    out = []
    for _ in range(n):
        qb = _rand_quat(rng)
        if t1 == "plane":
            if t2 == "mesh":
                ext = _rbound(t2, None)
            else:
                ext = float(Geom(t2, _pad(sizes[1] or SIZES[t2]), np.zeros(3), quat2mat(qb)).extent(np.array([[0, 0, -1.0]]))[0])
            z = ext * rng.uniform(0.4, 1.15)
            out.append(np.concatenate([[rng.uniform(-0.2, 0.2), rng.uniform(-0.2, 0.2), z], qb]))
        else:
            qa = _rand_quat(rng)
            d = rng.normal(size=3)
            d /= np.linalg.norm(d)
            r = (_rbound(t1, sizes[0]) + _rbound(t2, sizes[1])) * rng.uniform(0.15, 0.9)
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
