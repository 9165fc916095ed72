"""The CPU oracle's narrow phase against exact fp64 geometry (tests/narrow_phase_ref.py), for every geom type pair the compiler puts
in the pair list: seeded random poses around contact, at the model's sizes and at both ends of a +-30 % size range, and a named
catalogue of degenerate configurations (coincident centres, intersecting capsule cores, exact touch, aligned faces, edge-edge,
vertex-face, cylinders on a plane, deep penetration).

Rules, per pose:
- a contact exists exactly when the exact signed distance is below -band; within the band either answer is accepted;
- the deepest contact's dist equals the exact signed distance (analytic routines: 1e-9; GJK / EPA pairs: EPA_TOL); box-box
  accepts the routine's face preference, depth in [SAT, 1.05 SAT + 1e-5];
- every contact: dist <= 0, an orthonormal right-handed frame whose first row is the normal, pos within |dist| / 2 + tol of both
  surfaces (plane-capsule: of the plane and of the contact's end sphere); the deepest contact's normal points from geom1 to geom2
  (shifting geom2 by -dist along it separates the pair; box-box, whose clipped face manifold can miss the deepest incident vertex:
  the overlap along it is within the face-preference bound);
- at most 4 contacts for plane-box, plane-cylinder and plane-mesh, 8 for box-box, 2 for plane-capsule, 1 for every other pair.
"""
import numpy as np
import pytest

from tests import narrow_phase_ref as npr

# EPA stops when the support along the closest face's normal is within 1e-7 of the face, or when its polytope is full (96 vertices,
# 192 faces).  Polyhedral pairs converge: measured depth error <= 1.4e-15.  A curved surface needs more faces than that at deep
# penetration: the depth comes out short by up to 1 % of itself (5.9e-4 of 0.06 for two coincident cylinders, 6.9e-5 for random
# ellipsoid-ellipsoid poses), and the face normal is further off: along it up to 12 % of the depth is left unresolved (two coincident
# ellipsoids at different orientations).  Pairs with a curved geom get relative terms above those measured worst cases.
EPA_TOL = 1e-6
CURVED = {"sphere", "capsule", "ellipsoid", "cylinder"}
TOL_ANALYTIC = dict(band=1e-9, depth=1e-9, pos=1e-9, frame=1e-9, sep=1e-9)
TOL_GJK = dict(band=1e-7, depth=EPA_TOL, pos=1e-5, frame=1e-9, sep=EPA_TOL)
TOL_GJK_CURVED = dict(TOL_GJK, rel=0.015, sep_rel=0.15)
N_RANDOM_ANALYTIC, N_RANDOM_GJK = 300, 40


def _oracle(model):
    from oracle.pyoracle import Oracle
    from robosuite_b200.mjcf.compiler import pack_model

    return Oracle(pack_model(model))


def tolerances(pair):
    if pair in npr.ANALYTIC:
        return TOL_ANALYTIC
    return TOL_GJK_CURVED if CURVED & set(pair) else TOL_GJK


def run_oracle(model, o, qpos):
    """contacts of the scene at qpos: (geoms, [(dist, pos, frame)], geom id pairs)"""
    o.reset_data()
    o.qpos[:] = qpos
    o.forward()
    cs = o.contacts()
    return npr.geoms_of(model, o), [(c["dist"], c["pos"].copy(), c["frame"].copy()) for c in cs], [(c["geom1"], c["geom2"]) for c in cs]


def check_pose(pair, model, o, qpos):
    """failures of one pose, and the depth error of its deepest contact (None without a contact)"""
    geoms, cons, ids = run_oracle(model, o, qpos)
    A, B = geoms[:2]
    bad = []
    if any(g != (0, 1) for g in ids):
        bad.append("geom ids %s" % ids)
    extra = [np.asarray(c[2])[0] for c in cons]
    ref = npr.signed_distance(A, B, extra)
    bad += npr.check_contacts(pair, A, B, cons, ref, tolerances(pair))
    err = abs(min(c[0] for c in cons) - ref) if cons and pair != ("box", "box") else (0.0 if cons else None)
    return bad, err


def _catalogue_cases():
    return [pytest.param(pair, name, q, id="%s:%s" % (npr.pair_name(pair), name))
            for pair in npr.pair_types() for name, q, _ in npr.catalogue(pair)]


_MODELS = {}


def scene(pair, sizes=(None, None), meshes=("probe", "probe"), far=None):
    key = (pair, sizes, meshes, far)
    if key not in _MODELS:
        m = npr.compile_scene(npr.scene_xml(pair, sizes, meshes, far))
        assert m.npair == 1 and m.ngeom == (3 if far else 2)
        _MODELS[key] = (m, _oracle(m))
    return _MODELS[key]


@pytest.mark.parametrize("pair,name,qpos", _catalogue_cases())
def test_catalogue(pair, name, qpos):
    model, o = scene(pair)
    bad, _ = check_pose(pair, model, o, qpos)
    assert not bad, bad


@pytest.mark.parametrize("pair", npr.pair_types(), ids=npr.pair_name)
def test_random_poses(pair):
    n = N_RANDOM_ANALYTIC if pair in npr.ANALYTIC else N_RANDOM_GJK
    fails, worst, hits = [], 0.0, 0
    variants = [(1.0, (None, None))] + npr.size_variants(pair)
    for k, (scale, sizes) in enumerate(variants):
        model, o = scene(pair, sizes)
        for i, q in enumerate(npr.random_poses(pair, n if k == 0 else n // 4, seed=100 * k + 7)):
            bad, err = check_pose(pair, model, o, q)
            if err is not None:
                hits += 1
                worst = max(worst, err)
            if bad:
                fails.append((scale, i, bad))
    print("%s: %d poses with a contact, worst depth error %.3g" % (npr.pair_name(pair), hits, worst))
    assert hits >= n // 4, "too few poses in contact: %d" % hits
    assert not fails, (len(fails), fails[:5])
