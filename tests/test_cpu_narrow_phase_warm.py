"""CPU checks of the references test_gpu_narrow_phase_warm.py judges the warm-started narrow phase with (tests/narrow_phase_ref.py):
the hulls of HULL_SCENES (every point a vertex, ties in the mirrored 200-vertex hull), the CPU oracle against exact geometry on them
(as test_cpu_narrow_phase.py holds it on the probe), the core helpers against closed forms, and the hull-staging table of the phase
pipeline from its capacity formula."""
import numpy as np
import pytest

from tests import narrow_phase_ref as npr
from tests.test_cpu_narrow_phase import TOL_GJK, TOL_GJK_CURVED, run_oracle, scene

# hulls of 200+ vertices are judged like curved surfaces: EPA's 96-vertex polytope cannot resolve them at deep penetration.  Measured
# worst: 1.19e-3 short of 7.45e-2 (1.6 %) for the 3000- and 200-vertex hulls at coincident centres, above the curved pairs' 1 %.
TOL_LARGE_HULL = dict(TOL_GJK_CURVED, rel=0.025)


def hull_tolerances(meshes):
    return TOL_GJK if max(len(npr.HULLS[m]) for m in meshes) <= 100 else TOL_LARGE_HULL


@pytest.mark.parametrize("name", list(npr.HULLS))
def test_every_hull_point_is_a_vertex(name):
    model, _ = scene(("mesh", "mesh"), (None, None), (name, name))
    assert int(model.mesh_vertnum[0]) == len(npr.HULLS[name])


def test_mirrored_hull_has_ties_across_lanes():
    V = npr.HULLS["hull200"]
    for d in ([1.0, 0, 0], [0, 0, -1.0], [0.6, 0, 0.8]):
        s = V @ np.array(d)
        top = np.flatnonzero(s == s.max())
        assert len(top) == 2 and top[0] % 32 != top[1] % 32


def test_staging_table():
    """the phase pipeline's staging case of every hull scene from its capacity formula, and every case of convex_convex among them"""
    seen = set()
    for name, (meshes, far) in npr.HULL_SCENES.items():
        model, _ = scene(("mesh", "mesh"), (None, None), meshes, far)
        nv = [int(model.mesh_vertnum[model.geom_dataid[g]]) for g in range(2)]
        got = tuple(npr.staging_case(nv[0], nv[1], meshes[0] == meshes[1], npr.pipeline_stage_cap(list(model.mesh_vertnum), p))
                    for p in ("f32", "f64"))
        assert got == npr.HULL_STAGING[name], (name, got)
        seen |= set(got)
    assert seen == set(npr.STAGING_CASES)
    # the formulas at their ends: 56 KB caps, and a unit-queue area too small to stage
    assert npr.pipeline_stage_cap([5000, 5000], "f64") == 7168 and npr.pipeline_stage_cap([5000, 5000], "f32") == 14336
    assert npr.unit_stage_cap(npr.EPA_AREA_WORDS + 63) == 0 and npr.staging_case(10, 10, True, 0) == "neither"


@pytest.mark.parametrize("name", list(npr.HULL_SCENES))
def test_oracle_on_hulls(name):
    meshes, far = npr.HULL_SCENES[name]
    model, o = scene(("mesh", "mesh"), (None, None), meshes, far)
    Q, _, names = npr.hull_poses(meshes, 4, seed=31, tail=model.qpos0[14:])
    tol = hull_tolerances(meshes)
    fails, hits = [], 0
    for q, nm in zip(Q, names):
        geoms, cons, ids = run_oracle(model, o, q)
        A, B = geoms[:2]
        ref = npr.signed_distance(A, B, [np.asarray(c[2])[0] for c in cons])
        hits += bool(cons)
        bad = npr.check_contacts(("mesh", "mesh"), A, B, cons, ref, tol) + (["geom ids %s" % ids] if any(g != (0, 1) for g in ids) else [])
        if bad:
            fails.append((nm, bad))
    assert hits >= len(Q) // 3 and not fails, (hits, fails)


def test_core_helpers_closed_forms():
    I = np.eye(3)
    # point-point: the centre distance; the separation along the centre line is that distance, across it minus the offset
    A = npr.Geom("sphere", [0.03], [0, 0, 1.0], I)
    B = npr.Geom("sphere", [0.02], [0.1, 0.05, 1.0], I)
    assert A.radius == 0.03 and A.core().t == "point"
    assert abs(npr.core_distance(A, B) - np.hypot(0.1, 0.05)) < 1e-15
    assert abs(npr.separation_along(A.core(), B.core(), A.pos - B.pos) - np.hypot(0.1, 0.05)) < 1e-15
    # segment-box: a capsule lying 0.03 above a box's top face (half height 0.02), tilted so one end is lower
    box = npr.Geom("box", [0.1, 0.1, 0.02], [0, 0, 1.0], I)
    R = npr.quat2mat(npr.axq([0, 1, 0], np.pi / 2 - 0.1))  # segment along x, its +end dipping by 0.05 sin(0.1)
    cap = npr.Geom("capsule", [0.01, 0.05], [0, 0, 1.05], R)
    want = 0.03 - 0.05 * np.sin(0.1)
    assert abs(npr.core_distance(cap, box) - want) < 1e-9
    assert abs(npr.separation_along(cap.core(), box, [0, 0, 1.0]) - want) < 1e-12
    assert npr.separation_along(cap.core(), box, [1.0, 0, 0]) < 0  # a direction that does not separate
    # segment-segment crossing at a 0.02 offset: distance 0.02
    a = npr.Geom("capsule", [0.01, 0.05], [0, 0, 1.0], npr.quat2mat(npr.axq([0, 1, 0], np.pi / 2)))
    b = npr.Geom("capsule", [0.01, 0.05], [0, 0.02, 1.0], I)
    assert abs(npr.core_distance(a, b) - 0.02) < 1e-15
