"""The convex narrow phase as the phase pipeline (mode 1) and the unit queue (mode 2) run it: with the GJK warm start (each pair's
separating direction remembered in `gjk_cache`) and the hull staging of convex_convex, neither of which the fused kernel's
forward() has.  One environment per (pose, seed): a first step(1) creates the cache, a snapshot row gets the pose, zero velocity and
the seed in the pair's cache entry, restore(), and the next step(1) runs its narrow phase at that pose from that seed.  Its
contacts come from the contact export, the cache it leaves from a second snapshot.

Seeds per pose, and what must hold:
- zero: contacts bit-identical to forward()'s (the fused kernel), in both schedules: staging changes no value;
- |c|^2 just below the 1e-12 threshold, and entries with an inf, -inf or NaN component (mesh pairs): the zero seed's bits;
- the pose's own converged entry, a neighbouring pose's (1 mm / 1 degree away), its negation, two random directions at the pair's
  bounding scale, and for penetrating poses the entry of the pose moved apart along the centre line until it is 1 mm separated:
  the exact-geometry rules (no contact missing below -band, the deepest dist within gate + depth + rel |sd| of the exact signed
  distance, npr.check_contacts for normals and positions), and for polyhedral pairs with small hulls also the oracle gates of
  test_gpu_narrow_phase (F64_GATES / F32_GATES).  Curved pairs and the hulls of 200+ vertices are held to exact geometry only:
  their EPA depth depends on the simplex GJK hands over (test_cpu_narrow_phase.py).
- modes 1 and 2 bit-identical under every seed (their staging capacities differ).

The cache protocol, after the seeded substep: an entry is exactly zero where the contact came from EPA (pairs without a radius, and
sphere / capsule pairs whose cores overlap); every entry the substep wrote certifies that the cores are separated
(npr.separation_along >= -CERT_TOL) and is no shorter than the core distance (v is a point of the Minkowski difference); one written
along with a contact of a sphere / capsule pair is the core distance (to CORE_REL |v| + CERT_TOL); a pose without contact whose entry
kept its seed is not penetrating; a pose beyond the bounding spheres (culled) keeps its seed; a masked reset zeroes exactly the masked
environments' entries.

Staging case of each hull scene (npr.HULL_SCENES), per schedule and precision.  The pipeline's follows from its capacity formula; the
unit queue's from the workspace stride the library reports (2716 words, 3608 with the far hull: 756 / 1648 reals for hulls):
    scene                 pipeline f32 / f64     unit queue f32 / f64
    probe-hull200         both / both            both / both
    hull2000a-hull2000b   both / only A          neither / neither
    hull3000-hull200      both / only B          only B / only B
    hull3000-hull3000     only A / neither       neither / neither
    probe-probe           only A / only A        same hull / same hull
    probe-probe+far200    same hull / same hull  same hull / same hull
    hull200-hull200       only A / only A        only A / only A
(test_hull_staging_cases_reached asserts the pipeline's column and that the union is every case of convex_convex).

Packaged models (test_packaged_models_along_trajectories): the seven models in the library's default configuration (warm start on,
modes 1 and 2, f32 and f64) under scripted contact-rich actions; after each control step every convex pair within its bounding
spheres is judged at the device's own exported poses by the rules above (capped per family and step), with the counts of MIN_TRAJ.

Measured on an H100 80GB HBM3 (700 W power limit).  Every gate is the cold path's: no warm seed needed a looser one, except the fp32
capsule faults recorded in WARM_KNOWN (the known fp32 fault of DESIGN.md section 3, which warm starts reach more often).  Worst
difference of a seeded contact from the zero seed's, |d dist| / |d pos| / |d frame| (frames of coincident-centre poses have no
unique value, hence differences of 2):
    polyhedral probe pairs (box-mesh, mesh-mesh, probe-hull200)   f64 2.1e-17 / 2.2e-16 / 8.2e-16, f32 1.9e-8 / 1.2e-7 / 3.6e-7
    sphere-mesh, capsule-mesh                                     f64 2.1e-17 / 3.6e-15 / 3.3e-13, f32 7.5e-9 / 6.9e-6 / 4.2e-4
    cylinder-mesh                                                 f64 6.7e-8 / 1.5e-4 / 1.9e-3,   f32 5.0e-7 / 9.9e-4 / 9.8e-3
    other curved pairs (ellipsoid-*, cylinder-{cylinder, box}, capsule-{ellipsoid, cylinder, box}, sphere-ellipsoid)
                                                                  f64 up to 2.7e-4 / 5.0e-2,       f32 up to 4.5e-2 (WARM_KNOWN)
    hulls of 200-3000 vertices                                    up to 4.1e-4 / 3.8e-2 in both precisions (EPA's polytope)
The hull scenes through the fused kernel against the oracle: f64 at most 1.3e-16 / 2.4e-15 / 7.3e-14, f32 3.3e-7 / 7.0e-6 / 2.2e-4.
"""
import numpy as np
import pytest

from tests import narrow_phase_ref as npr
from tests.test_cpu_narrow_phase import scene, tolerances
from tests.test_cpu_narrow_phase_warm import hull_tolerances
from tests.test_gpu_narrow_phase import (F32_BAND, F32_GATES, F32_KNOWN_MISSES, F64_GATES, compare, device_contacts, family,
                                         oracle_results, pose_set)

pytestmark = pytest.mark.gpu

GJK_PAIRS = [p for p in npr.pair_types() if p not in npr.ANALYTIC]
SEEDS = ("subthreshold", "converged", "neighbour", "approach", "negated", "random0", "random1")
NONFINITE = {"inf": (np.inf, 0.3, 0.1), "-inf": (0.2, -np.inf, 0.5), "nan": (np.nan, 0.1, 0.2), "inf-inf": (np.inf, -np.inf, 0.0)}
CERT_TOL = {"f64": 1e-9, "f32": 1e-5}
CORE_REL = {"f64": 1e-5, "f32": 1e-3}
LARGE = 100  # hulls above this many vertices are judged against exact geometry only


def _np(t):
    return t.cpu().numpy().astype(np.float64)


def run_seeded(model, Q, seeds, prec, mode, pidx, reset_mask=None):
    """one substep per environment e at Q[e] from cache entry seeds[e] of pair pidx: (ncon, geom, dist, pos, frame), the entries
    after, and with reset_mask the entries after a masked reset"""
    import torch

    from robosuite_b200.engine import BatchedSim

    sim = BatchedSim(model, len(Q), precision=prec)
    try:
        dt = sim.dtype
        sim.set_mode(mode)
        sim.set_contact_export(True)
        sim.step(1)
        snap = sim.snapshot()
        snap.field("qpos").copy_(torch.as_tensor(Q, dtype=dt))
        snap.field("qvel").zero_()
        cache = snap.field("gjk_cache")
        cache.zero_()
        cache[:, 3 * pidx:3 * pidx + 3] = torch.as_tensor(np.asarray(seeds), dtype=dt)
        sim.restore(snap)
        sim.step(1)
        c = sim.contacts()
        after = sim.snapshot().field("gjk_cache")[:, 3 * pidx:3 * pidx + 3].cpu().numpy().copy()
        torch.cuda.synchronize()
        assert int(sim.warn.abs().max()) == 0
        dev = (c["ncon"].cpu().numpy().astype(int), c["geom"].cpu().numpy().astype(int), _np(c["dist"]), _np(c["pos"]),
               _np(c["frame"]).reshape(len(Q), -1, 3, 3))
        reset = None
        if reset_mask is not None:
            sim.reset(torch.as_tensor(reset_mask.astype(np.uint8), device=sim.torch_device))
            reset = sim.snapshot().field("gjk_cache")[:, 3 * pidx:3 * pidx + 3].cpu().numpy().copy()
            torch.cuda.synchronize()
        return dev, after, reset
    finally:
        sim.close()


def _take(dev, idx):
    return tuple(a[idx] for a in dev)


def _same_bits(a, b, e, f=None):
    """contacts of env e of `a` and env f of `b` bit-identical"""
    f = e if f is None else f
    n = int(a[0][e])
    if n != int(b[0][f]):
        return False
    return all(np.array_equal(x[e, :n], y[f, :n]) for x, y in zip(a[1:], b[1:]))


def _geoms(model, o, q):
    o.reset_data()
    o.qpos[:] = q
    o.forward()
    return npr.geoms_of(model, o)[:2]


def _move_b(q, dx, rot=None):
    q = q.copy()
    q[7:10] += dx
    if rot is not None:
        R = npr.quat2mat(q[10:14]) @ rot
        w = np.sqrt(max(1 + np.trace(R), 1e-300)) / 2
        q[10:14] = [w, (R[2, 1] - R[1, 2]) / (4 * w), (R[0, 2] - R[2, 0]) / (4 * w), (R[1, 0] - R[0, 1]) / (4 * w)]
    return q


def approach_pose(A, B, q, gap=1e-3):
    """q with geom B moved along the centre line until the pair is `gap` apart: the least shift t at which some direction of the
    20,000-direction set separates the pair by `gap` (bisection; any separating direction proves at least that distance)"""
    d = B.pos - A.pos
    d = d / np.linalg.norm(d) if np.linalg.norm(d) > 1e-9 else np.array([0, 0, 1.0])
    F = A.support(npr._DIRS) + B.support(-npr._DIRS)
    proj = npr._DIRS @ d
    lo, hi = 0.0, 1.0
    for _ in range(60):
        t = (lo + hi) / 2
        if (F - t * proj).min() < -gap:
            hi = t
        else:
            lo = t
    return _move_b(q, hi * d)


class Case:
    """one scene: model, pose set, references, the cached pair's index and its family"""

    def __init__(self, pair, meshes=("probe", "probe"), far=None, n_random=None, name=None):
        self.pair, self.meshes, self.far, self.id = pair, meshes, far, name or npr.pair_name(pair)
        self.model, self.o = scene(pair, (None, None), meshes, far)
        m = self.model
        self.pidx = 0
        if n_random is not None:
            self.Q, self.amb, self.names = npr.hull_poses(meshes, n_random, seed=31, tail=m.qpos0[14:])
            nv = [int(m.mesh_vertnum[m.geom_dataid[g]]) for g in range(2)]
            self.large = max(nv) > LARGE
        else:
            self.Q, self.amb, self.names = pose_set(pair)
            self.large = False
        self.ref = oracle_results(pair, self.Q, meshes=meshes, far=far)
        self.fam = "gjk_curved" if self.large else family(pair)
        self.exact_only = self.fam == "gjk_curved"
        self.geoms = [_geoms(m, self.o, q) for q in self.Q]
        self.ra_rb = self.geoms[0][0].radius + self.geoms[0][1].radius
        self.tols = hull_tolerances(meshes) if pair == ("mesh", "mesh") else tolerances(pair)


_CHECKED = {}


def exact_rules(case, prec, dev, e, i):
    """failures of env e of dev (pose i) against exact geometry"""
    ncon, _, dist, pos, frame = dev
    n = int(ncon[e])
    oc, sd = case.ref[i]
    gate = (F64_GATES if prec == "f64" else F32_GATES)[case.fam]
    band = case.tols["band"] if prec == "f64" else F32_BAND
    if prec == "f32" and case.names[i] in F32_KNOWN_MISSES.get(case.pair, ()) and case.meshes == ("probe", "probe"):
        return []
    bad = []
    if sd < -band and n == 0:
        bad.append("no contact at exact dist %.3g" % sd)
    if n == 0:
        return bad
    if abs(dist[e, :n].min() - sd) > gate[0] + case.tols["depth"] + case.tols.get("rel", 0.0) * abs(sd):
        bad.append("deepest dist %.9g vs exact %.9g" % (dist[e, :n].min(), sd))
    cons = [(dist[e, k], pos[e, k], frame[e, k]) for k in range(n)]
    key = (case.pair, case.meshes, prec, i, b"".join(np.asarray(c[k]).tobytes() for c in cons for k in range(3)))
    if key not in _CHECKED:
        t = case.tols
        tol = dict(t, band=band, depth=t["depth"] + gate[0], pos=t["pos"] + gate[1], frame=t["frame"] + gate[2], sep=t["sep"] + gate[0])
        A, B = case.geoms[i]
        _CHECKED[key] = npr.check_contacts(case.pair, A, B, cons, sd, tol)
    return bad + _CHECKED[key]


def _absent(s):
    """a seed the narrow phase treats as no remembered direction (b2s_collide.cuh warm_direction)"""
    return not np.isfinite(s).all() or float(np.dot(s, s)) <= 1e-12


_CORE = {}


def _core_distance(case, i):
    """the exact core distance at pose i (negative: the cores overlap), once per scene and pose"""
    key = (case.id, i)
    if key not in _CORE:
        _CORE[key] = npr.core_distance(*case.geoms[i])
    return _CORE[key]


def cache_protocol(case, prec, dev, after, seeds, poses, kinds):
    """failures (pose, seed kind, message) of the cache protocol: env e ran pose poses[e] from seeds[e] and left after[e]"""
    bad = []
    ncon = dev[0]
    for e, i in enumerate(poses):
        A, B = case.geoms[i]
        c, s = after[e], np.asarray(seeds[e], dtype=after.dtype)
        n = int(ncon[e])
        tag = (case.names[i], kinds[e])
        if prec == "f32" and case.names[i] in F32_KNOWN_MISSES.get(case.pair, ()) and case.meshes == ("probe", "probe"):
            continue
        kept = c.tobytes() == s.tobytes()
        # a contact came from EPA when the pair has no radius, or when its cores overlap (sphere / capsule pairs)
        epa = n and (case.ra_rb == 0 or _core_distance(case, i) < -CERT_TOL[prec])
        if epa and np.any(c != 0):
            bad.append(tag + ("contact from EPA but entry %s" % c,))
        if np.any(c != 0) and not kept:  # a kept seed may be a culled pair's, or a dismissal's (its own certificate)
            if not np.isfinite(c).all():
                bad.append(tag + ("non-finite entry %s" % c,))
                continue
            sep = npr.separation_along(A.core(), B.core(), c.astype(np.float64))
            if sep < -CERT_TOL[prec]:
                bad.append(tag + ("entry does not separate the cores: %.3g" % sep,))
            # every GJK-written v is a point of the Minkowski difference: never shorter than the core distance; with a contact of a
            # sphere / capsule pair GJK ran to convergence, so v is that distance
            v, cd = float(np.linalg.norm(c.astype(np.float64))), _core_distance(case, i)
            if v < cd - CERT_TOL[prec]:
                bad.append(tag + ("|v| %.9g below the core distance %.9g" % (v, cd),))
            if n and case.ra_rb > 0 and v - cd > CORE_REL[prec] * v + CERT_TOL[prec]:
                bad.append(tag + ("|v| %.9g vs core distance %.9g" % (v, cd),))
        if n == 0 and kept and not _absent(s):
            sd = case.ref[i][1]
            if sd < -(case.tols["band"] if prec == "f64" else F32_BAND):
                bad.append(tag + ("entry kept its seed without contact at exact dist %.3g" % sd,))
    return bad


def _rand_dirs(rng, k, scale):
    d = rng.normal(size=(k, 3))
    return scale * d / np.linalg.norm(d, axis=1, keepdims=True)


def run_case(case, prec):
    """section by section, both schedules; returns failures"""
    Q, n = case.Q, len(case.Q)
    rng = np.random.default_rng(11)
    scale = npr._rbound(case.pair[0], None, case.meshes[0]) + npr._rbound(case.pair[1], None, case.meshes[1])
    cold = device_contacts(case.model, Q, prec)
    # neighbour poses: B 1 mm along a random direction and turned 1 degree; approach poses for the penetrating ones
    Qn = np.array([_move_b(q, _rand_dirs(rng, 1, 1e-3)[0], npr.quat2mat(npr.axq(rng.normal(size=3), np.pi / 180))) for q in Q])
    band = case.tols["band"] if prec == "f64" else F32_BAND
    pen = [i for i in range(n) if case.ref[i][1] < -band]
    Qa = np.array([approach_pose(*case.geoms[i], Q[i]) for i in pen]).reshape(-1, Q.shape[1])
    mesh = "mesh" in case.pair
    sub, rand0, rand1 = _rand_dirs(rng, n, 9.9e-7), _rand_dirs(rng, n, scale), _rand_dirs(rng, n, scale)
    far_seed = _rand_dirs(rng, min(n, 8), scale)
    bad, res = [], {}
    worst = np.zeros(3)
    for mode in (1, 2):
        Z = np.concatenate([Q, Qn, Qa])
        zdev, zafter, _ = run_seeded(case.model, Z, np.zeros((len(Z), 3)), prec, mode, case.pidx)
        conv, neigh, appr = zafter[:n], zafter[n:2 * n], zafter[2 * n:]
        for e in range(n):
            if not _same_bits(zdev, cold, e):
                bad.append((mode, case.names[e], "zero", "zero seed differs from forward()"))
        bad += [(mode,) + b for b in cache_protocol(case, prec, _take(zdev, slice(0, n)), conv, np.zeros((n, 3)), range(n), ["zero"] * n)]
        seeds, poses, kinds = [], [], []

        def add(kind, idx, vals):
            for i, v in zip(idx, vals):
                seeds.append(v); poses.append(i); kinds.append(kind)

        add("subthreshold", range(n), sub)
        add("converged", range(n), conv)
        add("neighbour", range(n), neigh)
        add("approach", pen, appr)
        add("negated", range(n), -conv)
        add("random0", range(n), rand0)
        add("random1", range(n), rand1)
        if mesh:
            for k, v in NONFINITE.items():
                add(k, range(n), [v] * n)
        # culled: B beyond the bounding spheres, a random entry that must stay
        far_q = []
        for i in range(min(n, 8)):
            q = Q[i].copy()
            q[7:10] = q[0:3] + [1.5 * scale + 0.05, 0, 0]
            far_q.append(q)
        nfar = len(far_q)
        S = np.concatenate([np.array(seeds, dtype=np.float64), far_seed])
        P = np.concatenate([Q[np.array(poses)], np.array(far_q)])
        mask = (np.arange(len(P)) % 3 == 0)
        sdev, safter, sreset = run_seeded(case.model, P, S, prec, mode, case.pidx, reset_mask=mask)
        m = len(seeds)
        res[mode] = (sdev, safter, zdev, zafter)
        for e in range(m):
            i, kind = poses[e], kinds[e]
            if kind in NONFINITE or kind == "subthreshold":
                if not _same_bits(sdev, zdev, e, i):
                    bad.append((mode, case.names[i], kind, "differs from the zero seed"))
                continue
            if kind == "approach" and int(sdev[0][e]) == 0 and not (prec == "f32" and case.names[i] in F32_KNOWN_MISSES.get(case.pair, ())):
                bad.append((mode, case.names[i], kind, "no contact coming into contact (exact dist %.3g)" % case.ref[i][1]))
            if not _same_bits(sdev, zdev, e, i):  # the zero seed's contacts are forward()'s, which test_gpu_narrow_phase judges
                bad += [(mode, case.names[i], kind, b) for b in exact_rules(case, prec, sdev, e, i)]
            n0 = int(zdev[0][i])
            if n0 and int(sdev[0][e]) == n0:
                worst = np.maximum(worst, [np.abs(sdev[2][e, :n0] - zdev[2][i, :n0]).max(), np.abs(sdev[3][e, :n0] - zdev[3][i, :n0]).max(),
                                           np.abs(sdev[4][e, :n0] - zdev[4][i, :n0]).max()])
        if not case.exact_only:
            for kind in SEEDS:
                idx = [e for e in range(m) if kinds[e] == kind]
                if idx:
                    pi = [poses[e] for e in idx]
                    b, _ = compare(case.pair, prec, _take(sdev, np.array(idx)), [case.ref[i] for i in pi], [case.amb[i] for i in pi],
                                   [case.names[i] for i in pi], fam=case.fam, tols=case.tols)
                    bad += [(mode, x[0], kind, x[1]) for x in b]
        bad += [(mode,) + b for b in cache_protocol(case, prec, _take(sdev, slice(0, m)), safter[:m], S[:m], poses, kinds)]
        cast = S.astype(np.float32 if prec == "f32" else np.float64)
        for e in range(m, m + nfar):
            if not np.array_equal(safter[e], cast[e]) or int(sdev[0][e]) != 0:
                bad.append((mode, "far%d" % (e - m), "random", "culled pair changed its entry %s, seed %s" % (safter[e], cast[e])))
        if not (np.all(sreset[mask] == 0) and sreset[~mask].tobytes() == safter[~mask].tobytes()):
            bad.append((mode, "all", "all", "masked reset"))
    for e in range(len(res[1][0][0])):
        if not _same_bits(res[1][0], res[2][0], e):
            bad.append((2, "env%d" % e, "any", "modes 1 and 2 differ"))
    if res[1][1].tobytes() != res[2][1].tobytes():
        bad.append((2, "all", "any", "modes 1 and 2 leave different cache entries"))
    print("%s %s: worst difference from the zero seed |d dist| %.3g |d pos| %.3g |d frame| %.3g" % (case.id, prec, *worst))
    return bad


# warm-start faults these tests found that this module does not fix: (scene, precision) -> {(pose, seed kind)}.  Each must still fail
# (a fix shows up here), and nothing else may.  All are fp32 capsule pairs, and all are the known fp32 fault of DESIGN.md section 3
# (F32_KNOWN_MISSES): from these starting directions the fp32 GJK stops with |v| at the rounding of metre-scale support points, above
# its overlap test, on a segment core that overlaps the other core.  It then reports the cores separated: the contact's depth is
# about -(ra + rb) and its normal is the direction of a rounding-level v (measured: depth off by up to 4.5e-2, normals that leave
# up to 5.7e-2 of overlap beyond the depth, entries that fail the separation certificate by up to 8.5e-2).  The zero seed reaches it for
# capsule-ellipsoid random17 / random21 (their contacts are forward()'s: test_gpu_narrow_phase holds those within its gates).
WARM_KNOWN = {
    ('capsule-box', 'f32'): {
        ('concentric_rotated', 'random0')},
    ('capsule-cylinder', 'f32'): {
        ('random20', 'random0'), ('random21', 'random0'), ('random26', 'negated'), ('random6', 'converged')},
    ('capsule-ellipsoid', 'f32'): {
        ('random17', 'approach'), ('random17', 'converged'), ('random17', 'random0'), ('random17', 'random1'), ('random17',
        'subthreshold'), ('random17', 'zero'), ('random2', 'converged'), ('random2', 'random1'), ('random21', 'approach'),
        ('random21', 'converged'), ('random21', 'neighbour'), ('random21', 'random0'), ('random21', 'random1'), ('random21',
        'subthreshold'), ('random21', 'zero'), ('random28', 'approach'), ('random28', 'random0'), ('random44', 'random1'),
        ('random47', 'converged')},
}


# failures no WARM_KNOWN entry covers: the bit-identity claims hold at every pose
BIT_IDENTITY = ("zero seed differs from forward()", "differs from the zero seed", "modes 1 and 2")


def _judge(scene_id, prec, bad):
    for b in bad:
        print("WARM-FAIL %s %s %s %s: %s" % (scene_id, prec, b[1], b[2], b[3]))
    known = WARM_KNOWN.get((scene_id, prec), set())
    new = [b for b in bad if (b[1], b[2]) not in known or b[3].startswith(BIT_IDENTITY)]
    gone = known - {(b[1], b[2]) for b in bad}
    assert not new and not gone, (len(new), new[:8], sorted(gone))


@pytest.mark.parametrize("prec", ["f64", "f32"])
@pytest.mark.parametrize("pair", GJK_PAIRS, ids=npr.pair_name)
def test_warm_start_pose_by_pose(pair, prec):
    _judge(npr.pair_name(pair), prec, run_case(Case(pair), prec))


def _hull_case(name):
    meshes, far = npr.HULL_SCENES[name]
    return Case(("mesh", "mesh"), meshes, far, n_random=8, name=name)


@pytest.mark.parametrize("prec", ["f64", "f32"])
@pytest.mark.parametrize("name", list(npr.HULL_SCENES))
def test_warm_start_hulls(name, prec):
    _judge(name, prec, run_case(_hull_case(name), prec))


@pytest.mark.parametrize("prec", ["f64", "f32"])
@pytest.mark.parametrize("name", list(npr.HULL_SCENES))
def test_hulls_cold_fused(name, prec):
    """the hull scenes through the fused kernel, as test_gpu_narrow_phase judges the catalogue's pairs"""
    case = _hull_case(name)
    bad, worst = compare(case.pair, prec, device_contacts(case.model, case.Q, prec), case.ref, case.amb, case.names, fam=case.fam, tols=case.tols)
    print("%s %s: worst |d dist| %.3g |d pos| %.3g |d frame| %.3g" % (name, prec, *worst))
    assert not bad, (len(bad), bad[:6], worst)


def test_hull_staging_cases_reached(capfd, monkeypatch):
    """the staging case of every hull scene per schedule and precision: the pipeline's from its capacity formula, the unit queue's
    from the workspace stride it reports; together they reach every case of convex_convex"""
    import torch

    from robosuite_b200.engine import BatchedSim

    monkeypatch.setenv("B2S_VERBOSE", "1")
    seen = set()
    for name, (meshes, far) in npr.HULL_SCENES.items():
        model, _ = scene(("mesh", "mesh"), (None, None), meshes, far)
        nv = [int(model.mesh_vertnum[model.geom_dataid[g]]) for g in range(2)]
        for k, prec in enumerate(("f32", "f64")):
            pipe = npr.staging_case(nv[0], nv[1], meshes[0] == meshes[1], npr.pipeline_stage_cap(list(model.mesh_vertnum), prec))
            assert pipe == npr.HULL_STAGING[name][k]
            sim = BatchedSim(model, 2, precision=prec)
            try:
                capfd.readouterr()
                sim.set_mode(2)
                sim.step(1)
                torch.cuda.synchronize()
            finally:
                sim.close()
            err = capfd.readouterr().err
            # the stride is only reported by the library's B2S_VERBOSE line "... <k> words/warp ..."
            words = [ln.split("words/warp")[0].split(",")[-1] for ln in err.splitlines() if "unit-queue" in ln and "words/warp" in ln]
            assert words, "the unit queue's B2S_VERBOSE line (its workspace stride) is missing: %r" % err
            stride = int(words[-1])
            unit = npr.staging_case(nv[0], nv[1], meshes[0] == meshes[1], npr.unit_stage_cap(stride))
            with capfd.disabled():
                print("%s %s: pipeline %s, unit queue %s (stride %d words)" % (name, prec, pipe, unit, stride))
            seen |= {pipe, unit}
    assert seen == set(npr.STAGING_CASES), sorted(set(npr.STAGING_CASES) - seen)


# ------------------------------------------------------------------------------------------------ packaged models along trajectories
PACKAGED = [("Lift", "Panda"), ("Stack", "Panda"), ("Door", "Panda"), ("NutAssemblyRound", "Panda"), ("PickPlace", "Panda"),
            ("Lift", "Sawyer"), ("Stack", "Sawyer")]
N_TRAJ, STEPS_TRAJ, FROM_TRAJ = 8, 12, 5  # environments and control steps per handle; pairs are judged from this step on
CAP_TRAJ = 2  # judged pairs per family, control step and handle (pairs with a contact first): the fp64 reference costs ~0.3 s a pair
# least (judged pairs, judged contacts) per family over both schedules and precisions, half of what these trajectories give on an H100
# (56 pairs within their bounding spheres for every family listed; the few cylinder-box pairs of the Panda models other than Door
# never come that close).  Only box-mesh pairs (finger pads on the objects, PickPlace's objects in
# their bin) come into contact: the other families are robot-internal or door pairs that these scripted actions bring close but
# never into contact, where the judgement is that no contact is missing.  Sawyer's cylinder-cylinder pairs, the pair of the known
# fp32 fault (F32_KNOWN_MISSES), are among them: the fault does not show up on a packaged model here.
_PANDA = {"mesh-mesh": (28, 0), "cylinder-mesh": (28, 0)}
MIN_TRAJ = {"Lift_Panda": dict(_PANDA, **{"box-mesh": (28, 1)}), "Stack_Panda": dict(_PANDA, **{"box-mesh": (28, 1)}),
            "Door_Panda": dict(_PANDA, **{"box-mesh": (28, 0), "cylinder-box": (28, 0), "cylinder-cylinder": (28, 0)}),
            "NutAssemblyRound_Panda": dict(_PANDA, **{"box-mesh": (28, 4)}), "PickPlace_Panda": dict(_PANDA, **{"box-mesh": (28, 28)}),
            "Lift_Sawyer": {"cylinder-box": (28, 0), "cylinder-cylinder": (28, 0)},
            "Stack_Sawyer": {"cylinder-box": (28, 0), "cylinder-cylinder": (28, 0)}}
_TRAJ = {}


def _convex_pairs(m):
    """(g1, g2, family name) of every GJK pair of the model, the geoms in the narrow phase's order (lower type first)"""
    inv = {v: k for k, v in npr.TYPES.items()}
    out = []
    for g1, g2 in np.asarray(m.pair_geom).reshape(-1, 2):
        g1, g2 = int(g1), int(g2)
        if m.geom_type[g1] > m.geom_type[g2]:
            g1, g2 = g2, g1
        pair = (inv[int(m.geom_type[g1])], inv[int(m.geom_type[g2])])
        if "plane" not in pair and pair not in npr.ANALYTIC:
            out.append((g1, g2, pair))
    return out


def _world_geom(m, g, pos, mat):
    inv = {v: k for k, v in npr.TYPES.items()}
    t = inv[int(m.geom_type[g])]
    vert = None
    if t == "mesh":
        k = int(m.geom_dataid[g])
        a, n = int(m.mesh_vertadr[k]), int(m.mesh_vertnum[k])
        vert = np.array(m.mesh_vert[a:a + n], dtype=np.float64)
    return npr.Geom(t, m.geom_size[g], pos, mat, vert)


def judge_pair(m, g1, g2, pair, prec, pos, mat, cons):
    """failures of one convex pair at the device's poses (cast to fp64) and its contacts [(dist, pos, frame)]"""
    A, B = _world_geom(m, g1, pos[g1], mat[g1]), _world_geom(m, g2, pos[g2], mat[g2])
    key = (prec, A.pos.tobytes(), A.mat.tobytes(), B.pos.tobytes(), B.mat.tobytes(), repr(cons))
    if key in _TRAJ:
        return _TRAJ[key]
    large = max((len(G.vert) for G in (A, B) if G.vert is not None), default=0) > LARGE
    fam = "gjk_curved" if large else family(pair)
    t = hull_tolerances(("hull200",)) if large else tolerances(pair)
    gate = (F64_GATES if prec == "f64" else F32_GATES)[fam]
    band = t["band"] if prec == "f64" else F32_BAND
    sd = npr.signed_distance(A, B, [np.asarray(c[2])[0] for c in cons])
    bad = []
    if sd < -band and not cons:
        bad.append("no contact at exact dist %.3g" % sd)
    if cons:
        if abs(min(c[0] for c in cons) - sd) > gate[0] + t["depth"] + t.get("rel", 0.0) * abs(sd):
            bad.append("deepest dist %.9g vs exact %.9g" % (min(c[0] for c in cons), sd))
        tol = dict(t, band=band, depth=t["depth"] + gate[0], pos=t["pos"] + gate[1], frame=t["frame"] + gate[2], sep=t["sep"] + gate[0])
        bad += npr.check_contacts(pair, A, B, cons, sd, tol)
    _TRAJ[key] = bad
    return bad


def rollout_checks(task, robot, prec, mode):
    """judge the convex pairs of a scripted contact-rich rollout in the library's default configuration: after every control step the
    last substep's contacts and its exported geom_xpos / geom_xmat, which are the narrow phase's inputs (export_kinematics writes the
    poses phase 0 computed for that substep's narrow phase).  Returns (failures, judged pairs per family, judged contacts per family)"""
    import torch

    from tests.schedules import make_env, random_actions

    env = make_env(task, N_TRAJ, mode, 7, robots=robot, precision=prec, contact_queries=True, data_queries=True)
    sim, m = env.sim, env.sim.model
    pairs = _convex_pairs(m)
    rb = np.asarray(m.geom_rbound, dtype=np.float64)
    acts = random_actions(env, STEPS_TRAJ)
    acts[:, :, -1] = 1.0  # gripper closing
    acts[1:, : N_TRAJ // 2, :3] = torch.as_tensor([0.0, 0.0, -1.0], dtype=acts.dtype, device=acts.device)  # half the arms push down
    bad, judged, contacts = [], {}, {}
    try:
        for t in range(STEPS_TRAJ):
            env.step(acts[t])
            if t < FROM_TRAJ:
                continue
            c = sim.contacts()
            torch.cuda.synchronize()
            ncon, geom, dist = c["ncon"].cpu().numpy(), c["geom"].cpu().numpy(), _np(c["dist"])
            cpos, cfr = _np(c["pos"]), _np(c["frame"]).reshape(N_TRAJ, -1, 3, 3)
            xpos, xmat = _np(sim.data.geom_xpos), _np(sim.data.geom_xmat).reshape(N_TRAJ, -1, 3, 3)
            warn = sim.warn.cpu().numpy()
            todo = {}
            for e in range(N_TRAJ):
                if warn[e] & 4:  # contact overflow: the kept contacts are not all of them
                    continue
                for g1, g2, pair in pairs:
                    if np.linalg.norm(xpos[e, g1] - xpos[e, g2]) > rb[g1] + rb[g2]:
                        continue
                    cons = [(dist[e, k], cpos[e, k], cfr[e, k]) for k in range(int(ncon[e])) if tuple(geom[e, k]) == (g1, g2)]
                    todo.setdefault(pair, []).append((not cons, e, g1, g2, cons))
            for pair, items in todo.items():
                for _, e, g1, g2, cons in sorted(items, key=lambda x: (x[0], x[1], x[2], x[3]))[:CAP_TRAJ]:
                    judged[pair] = judged.get(pair, 0) + 1
                    contacts[pair] = contacts.get(pair, 0) + bool(cons)
                    for b in judge_pair(m, g1, g2, pair, prec, xpos[e], xmat[e], cons):
                        bad.append((t, e, m.names["geom"][g1] if "geom" in m.names else g1, m.names["geom"][g2] if "geom" in m.names else g2, b))
    finally:
        env.close()
    return bad, judged, contacts


@pytest.mark.parametrize("task,robot", PACKAGED, ids=["%s_%s" % p for p in PACKAGED])
def test_packaged_models_along_trajectories(task, robot):
    """modes 1 and 2, f32 and f64: every judged convex pair by the rules of the pose-by-pose test, every family of the model judged,
    and at least MIN_TRAJ judged pairs and contacts per family"""
    name = "%s_%s" % (task, robot)
    bad, judged, contacts = [], {}, {}
    for prec in ("f64", "f32"):
        for mode in (1, 2):
            b, j, c = rollout_checks(task, robot, prec, mode)
            bad += [(prec, mode) + x for x in b]
            for k, v in j.items():
                judged[k] = judged.get(k, 0) + v
            for k, v in c.items():
                contacts[k] = contacts.get(k, 0) + v
    print("TRAJ %s judged pairs %s contacts %s" % (name, {npr.pair_name(k): v for k, v in judged.items()},
                                                   {npr.pair_name(k): v for k, v in contacts.items()}))
    got = {npr.pair_name(k): (judged[k], contacts.get(k, 0)) for k in judged}
    assert set(got) == set(MIN_TRAJ[name]), (sorted(got), sorted(MIN_TRAJ[name]))
    short = {f: got[f] for f, (j, c) in MIN_TRAJ[name].items() if got[f][0] < j or got[f][1] < c}
    assert not short, short
    assert not bad, (len(bad), bad[:8])
