"""The device narrow phase, pose by pose, against the fp64 CPU oracle and exact geometry (tests/narrow_phase_ref.py), for every geom type
pair the compiler puts in the pair list.  One environment per pose (the random poses and the degenerate catalogue of
test_cpu_narrow_phase.py), one `BatchedSim.forward()` (the fused kernel, with export), then contact by contact: ncon, geom ids and
order, dist, pos and frame.

- f64: the same routines in the same precision as the oracle: agreement at rounding level (F64_GATES; curved GJK pairs at the
  level of GJK's convergence test).
- f32: gates per routine family (F32_GATES).  Worst |d dist| / |d pos| / |d frame| against the oracle over this file's poses,
  measured on an H100 80GB HBM3 (700 W power limit):
    analytic routines                        1.6e-7 / 5.9e-7 / 3.7e-5
    GJK / EPA, polyhedral pairs              8.0e-8 / 1.1e-7 / 2.0e-6
    GJK / EPA, pairs with a curved geom      2.0e-5 / 4.9e-4 / 3.8e-2  (the fp32 GJK stops at 32 iterations on grazing pairs)
  and in f64, curved GJK / EPA pairs: 1.5e-7 / 3.8e-5 / 4.6e-3, every other pair at most 2.2e-16 / 4.4e-16 / 2.1e-14.
  Poses whose oracle contact count differs from the device's are only accepted when a contact or the exact signed distance lies
  within F32_BAND of zero (knife-edge contacts).  Positions and frames are not compared where they have no unique value (coincident
  centres, intersecting capsule cores, two equally good reference faces); there the depth is held to the exact reference.
- Broad phase: every pose whose exact signed distance is below -F32_BAND has a contact, in both precisions.  This covers the
  bounding-sphere cull and `obb_overlap` for every type, the plane test included.
- Per-environment sizes: `model_override("geom_size", g)` gives both geoms of a pair different sizes per environment (the model's,
  x0.7 and x1.3), and each environment is compared with an oracle compiled at its sizes.  This runs `geom_size_of` and the bounding
  radius / box of the set-constants pass, which no packaged model exercises for capsules and ellipsoids.
- Schedules: one scene with a one-hinge arm and probes of every primitive type resting on a plane and on each other, JOINT_TORQUE with
  zero actions: two control steps from the same states in modes 0, 1 and 2 (controller in the tail kernel, no GJK warm start) give
  bit-identical qpos and qvel.  The pipeline's and the unit queue's thread-per-pair analytic role runs sphere, capsule and cylinder
  pairs here, which no packaged model puts in contact.
"""
import os

import numpy as np
import pytest

from tests import narrow_phase_ref as npr
from tests.test_cpu_narrow_phase import CURVED, scene, tolerances

pytestmark = pytest.mark.gpu

N_RANDOM_ANALYTIC, N_RANDOM_GJK = 192, 48
F32_BAND = 1e-4
# fp32 faults these tests found that this module does not fix, by pose: each must still be a missing contact (a fix shows up here).
# Two crossed cylinders 5 mm deep: the fp32 GJK stops with the origin on a face of its simplex, |v| at the rounding of metre-scale
# support points (above its 1e-8 overlap test), and reports the cores separated.  Treating such a core distance as an overlap gives
# the right contact, but the benchmarked Lift model's cylinder-box and mesh pairs reach the same branch and their results move.
F32_KNOWN_MISSES = {("cylinder", "cylinder"): {"crossed"}}
# f64 vs the oracle: (dist, pos, frame) absolute.  Analytic and polyhedral pairs at rounding level; curved GJK pairs at GJK's own
# convergence level (it stops once |v|^2 progresses by less than 1e-12 of itself; device and oracle round differently, so they may
# stop an iteration apart, which moves a normal of a curved surface by far more than one rounding)
F64_GATES = {"analytic": (1e-8, 1e-8, 1e-8), "gjk": (1e-8, 1e-8, 1e-8), "gjk_curved": (1e-6, 1e-4, 1e-2)}
# f32 vs the fp64 oracle: (dist, pos, frame) absolute, per routine family, about 5x the measured worst cases (module docstring)
F32_GATES = {"analytic": (2e-6, 5e-6, 3e-4), "gjk": (1e-6, 2e-6, 5e-5), "gjk_curved": (1e-4, 2e-3, 0.1)}


def family(pair):
    if pair in npr.ANALYTIC:
        return "analytic"
    return "gjk_curved" if CURVED & set(pair) else "gjk"


def pose_set(pair):
    """(qpos [n, nq], ambiguous-normal flags [n], names)"""
    n = N_RANDOM_ANALYTIC if pair in npr.ANALYTIC else N_RANDOM_GJK
    Q = list(npr.random_poses(pair, n, seed=17))
    amb = [False] * n
    names = ["random%d" % i for i in range(n)]
    for name, q, a in npr.catalogue(pair):
        Q.append(q); amb.append(a); names.append(name)
    return np.array(Q), amb, names


_REF = {}


def oracle_results(pair, Q, sizes_of=lambda i: (None, None)):
    """per pose: (oracle contacts [(dist, pos, frame, g1, g2)], exact signed distance); cached per pair and size set"""
    out = []
    for i, q in enumerate(Q):
        sizes = sizes_of(i)
        key = (pair, sizes, q.tobytes())
        if key not in _REF:
            model, o = scene(pair, sizes)
            o.reset_data()
            o.qpos[:] = q
            o.forward()
            cs = [(c["dist"], c["pos"].copy(), c["frame"].copy(), c["geom1"], c["geom2"]) for c in o.contacts()]
            A, B = npr.geoms_of(model, o)
            _REF[key] = (cs, npr.signed_distance(A, B, [c[2][0] for c in cs]))
        out.append(_REF[key])
    return out


def device_contacts(model, Q, prec, sizes=None):
    """forward() of one environment per pose; sizes: {geom id: [n, 3] array} per-environment geom sizes"""
    import torch

    from robosuite_b200.engine import BatchedSim

    sim = BatchedSim(model, len(Q), precision=prec)
    try:
        dt = sim.dtype
        if sizes:
            for g, s in sizes.items():
                sim.model_override("geom_size", g).copy_(torch.as_tensor(s, dtype=dt))
            sim.set_const()
        sim.qpos.copy_(torch.as_tensor(Q, dtype=dt))
        sim.forward()
        torch.cuda.synchronize()
        assert int(sim.warn.abs().max()) == 0
        get = lambda a: a.cpu().numpy().astype(np.float64)
        return (sim.ncon.cpu().numpy().astype(int), sim.contact_geom.cpu().numpy().astype(int), get(sim.contact_dist),
                get(sim.contact_pos), get(sim.contact_frame).reshape(len(Q), -1, 3, 3))
    finally:
        sim.close()


def compare(pair, prec, dev, ref, amb, names):
    """failures, and the worst (dist, pos, frame) differences"""
    ncon, geom, dist, pos, frame = dev
    worst = np.zeros(3)
    bad = []
    gate = (F64_GATES if prec == "f64" else F32_GATES)[family(pair)]
    band = tolerances(pair)["band"] if prec == "f64" else F32_BAND
    for e, (oc, sd) in enumerate(ref):
        n = int(ncon[e])
        if prec == "f32" and names[e] in F32_KNOWN_MISSES.get(pair, ()):
            if n != 0 or len(oc) == 0 or sd > -band:
                bad.append((names[e], "known fp32 miss changed: ncon %d, oracle %d, exact dist %.3g" % (n, len(oc), sd)))
            continue
        if sd < -band and n == 0:
            bad.append((names[e], "no contact at exact dist %.3g" % sd))
        if n != len(oc):
            edge = abs(sd) < band or any(abs(c[0]) < band for c in oc) or any(abs(d) < band for d in dist[e, :n])
            if prec == "f64" or not edge:
                bad.append((names[e], "ncon %d vs oracle %d (exact dist %.3g)" % (n, len(oc), sd)))
            continue
        if [tuple(g) for g in geom[e, :n]] != [(c[3], c[4]) for c in oc]:
            bad.append((names[e], "geom ids"))
        for k, c in enumerate(oc):
            # an ambiguous pose's deep EPA result depends on the polytope's path: its depth is held to the exact reference instead
            err = np.array([0.0 if amb[e] and family(pair) == "gjk_curved" else abs(dist[e, k] - c[0]), 0.0 if amb[e] else np.abs(pos[e, k] - c[1]).max(),
                            0.0 if amb[e] else np.abs(frame[e, k] - c[2]).max()])
            worst = np.maximum(worst, err)
            if (err > gate).any():
                bad.append((names[e], "contact %d: |d dist| %.3g |d pos| %.3g |d frame| %.3g" % (k, *err)))
        if n and (prec == "f32" or amb[e]) and pair != ("box", "box"):
            # the deepest contact against exact geometry too (the oracle's own agreement is test_cpu_narrow_phase's)
            tol = gate[0] + tolerances(pair)["depth"] + tolerances(pair).get("rel", 0.0) * abs(sd)
            if abs(dist[e, :n].min() - sd) > tol:
                bad.append((names[e], "deepest dist %.9g vs exact %.9g" % (dist[e, :n].min(), sd)))
    return bad, worst


@pytest.mark.parametrize("prec", ["f64", "f32"])
@pytest.mark.parametrize("pair", npr.pair_types(), ids=npr.pair_name)
def test_narrow_phase_matches_oracle_and_exact_geometry(pair, prec):
    model, _ = scene(pair)
    Q, amb, names = pose_set(pair)
    ref = oracle_results(pair, Q)
    assert sum(1 for oc, _ in ref if oc) >= len(Q) // 4  # the pose set is about contacts
    bad, worst = compare(pair, prec, device_contacts(model, Q, prec), ref, amb, names)
    print("%s %s: worst |d dist| %.3g |d pos| %.3g |d frame| %.3g" % (npr.pair_name(pair), prec, *worst))
    assert not bad, (len(bad), bad[:6], worst)


SIZED_PAIRS = [("plane", "sphere"), ("plane", "capsule"), ("plane", "ellipsoid"), ("plane", "cylinder"), ("plane", "box"),
               ("sphere", "capsule"), ("sphere", "cylinder"), ("capsule", "capsule"), ("capsule", "ellipsoid"),
               ("ellipsoid", "cylinder"), ("sphere", "box"), ("box", "box")]


@pytest.mark.parametrize("prec", ["f64", "f32"])
@pytest.mark.parametrize("pair", SIZED_PAIRS, ids=npr.pair_name)
def test_per_environment_sizes(pair, prec):
    variants = [(1.0, (None, None))] + npr.size_variants(pair)
    n0 = 48 if pair in npr.ANALYTIC else 16
    Q, sizes_per_env, amb, names = [], [], [], []
    for scale, sizes in variants:
        for i, q in enumerate(npr.random_poses(pair, n0, seed=23, sizes=sizes)):
            Q.append(q); sizes_per_env.append(sizes); amb.append(False); names.append("x%g/%d" % (scale, i))
    Q = np.array(Q)
    model, _ = scene(pair)
    dev_sizes = {}
    for g, t in enumerate(pair):
        if t == "plane":
            continue
        arr = np.tile(np.array(model.geom_size[g], dtype=np.float64), (len(Q), 1))
        for e, s in enumerate(sizes_per_env):
            if s[g] is not None:
                arr[e, :len(s[g])] = s[g]
        dev_sizes[g] = arr
    ref = oracle_results(pair, Q, lambda i: sizes_per_env[i])
    bad, worst = compare(pair, prec, device_contacts(model, Q, prec, dev_sizes), ref, amb, names)
    print("%s %s per-env sizes: worst |d dist| %.3g |d pos| %.3g |d frame| %.3g" % (npr.pair_name(pair), prec, *worst))
    assert not bad, (len(bad), bad[:6], worst)


# ------------------------------------------------------------------------------------------------ schedules
_QX = "0.70710678118654757 0 0.70710678118654757 0"  # local z along world x
_PROBES = [  # (type, size, pos, quat): resting on the plane (0.2 mm deep) and on each other (0.5-1.6 mm)
    ("box", "0.05 0.04 0.02", (0.8, 0, 0.0198), None),
    ("sphere", "0.03", (0.8, 0, 0.0693), None),  # on the box
    ("capsule", "0.02 0.06", (0.8, 0.0595, 0.0198), _QX),  # against the box's side
    ("cylinder", "0.03 0.05", (0.5, 0.2, 0.0498), None),  # upright
    ("capsule", "0.02 0.06", (0.5, 0.2, 0.1193), _QX),  # lying across the cylinder's cap
    ("cylinder", "0.03 0.05", (0.4, -0.1, 0.0298), _QX),  # lying
    ("sphere", "0.03", (0.4, -0.041, 0.0298), None),  # against the lying cylinder's side
    ("ellipsoid", "0.05 0.03 0.02", (0.3, 0.2, 0.0198), None),
    ("box", "0.05 0.04 0.02", (0.3, 0.2, 0.0591), None),  # on the ellipsoid
    ("sphere", "0.03", (0.376, 0.2, 0.0298), None),  # against the ellipsoid's tip
]  # ten free bodies: the engine takes at most 64 dofs


def _schedule_scene():
    probes = "".join('<body pos="%g %g %g"%s><freejoint/><geom type="%s" size="%s"/></body>'
                     % (*p, ' quat="%s"' % q if q else "", t, s) for t, s, p, q in _PROBES)
    return ('<mujoco><option timestep="0.002" cone="elliptic"/><worldbody><geom type="plane" size="2 2 0.1"/>'
            '<body name="robot0_base" pos="0 0 0.6"><site name="robot0_right_center"/>'
            '<body name="robot0_link1"><joint name="robot0_joint1" type="hinge" axis="0 1 0" damping="0.5"/>'
            '<geom type="capsule" size="0.02 0.1" pos="0.1 0 0" quat="%s" mass="0.5"/>'
            '<site name="gripper0_right_grip_site" pos="0.2 0 0"/></body></body>%s</worldbody>'
            '<actuator><motor name="robot0_torq_j1" joint="robot0_joint1" ctrlrange="-10 10"/></actuator></mujoco>' % (_QX, probes))


def _schedule_run(model, q, mode, steps=2):
    import torch

    from robosuite_b200 import controller_config as cc
    from robosuite_b200.engine import BatchedSim, CtrlCfg

    os.environ["B2S_NO_GJK_CACHE"] = "1"
    os.environ["B2S_CTRL_SPLIT"] = "0"
    try:
        sim = BatchedSim(model, len(q), precision="f32", maxcon=64, maxefc=256)  # 21 resting contacts, ~20 analytic candidates
        cfg = {"type": "BASIC", "body_parts": {"arms": {"right": cc.load_part_controller_config("JOINT_TORQUE")}}}
        sim.ctrl_config(cc.resolve(model, cfg, CtrlCfg))
        sim.set_export(False)
        sim.set_mode(mode)
        sim.qpos.copy_(torch.as_tensor(q, dtype=torch.float32))
        sim.forward()
        sim.ctrl_reset()
        act = torch.zeros((len(q), 2), dtype=torch.float32, device=sim.torch_device)
        for _ in range(steps):
            sim.env_step(act, 25)
        torch.cuda.synchronize()
        assert int(sim.warn.abs().max()) == 0
        out = sim.qpos.cpu().numpy().copy(), sim.qvel.cpu().numpy().copy()
        sim.close()
        return out
    finally:
        os.environ.pop("B2S_NO_GJK_CACHE", None)
        os.environ.pop("B2S_CTRL_SPLIT", None)


def test_schedules_bit_exact_on_primitive_contacts():
    """modes 0 (fused), 1 (phase pipeline) and 2 (unit queue) on a scene whose contacts are sphere / capsule / ellipsoid / cylinder /
    box pairs: bit-identical qpos and qvel after two control steps (50 substeps)"""
    from oracle.pyoracle import Oracle
    from robosuite_b200.mjcf.compiler import pack_model

    model = npr.compile_scene(_schedule_scene())
    rng = np.random.default_rng(5)
    n = 16
    q = np.tile(model.qpos0, (n, 1))
    q[:, 1::7] += rng.uniform(-2e-4, 2e-4, size=q[:, 1::7].shape)  # free-joint x / y / z of every probe (qpos[0] is the hinge)
    q[:, 2::7] += rng.uniform(-2e-4, 2e-4, size=q[:, 2::7].shape)
    q[:, 3::7] += rng.uniform(-2e-4, 1e-4, size=q[:, 3::7].shape)
    q[:, 0] = rng.uniform(-0.5, 0.5, n)
    o = Oracle(pack_model(model))
    o.qpos[:] = q[0]
    o.forward()
    types = {tuple(sorted((int(model.geom_type[c["geom1"]]), int(model.geom_type[c["geom2"]])))) for c in o.contacts()}
    want = {(0, 2), (0, 3), (0, 4), (0, 5), (0, 6), (2, 6), (3, 6), (3, 5), (2, 4), (2, 5), (4, 6)}
    assert want <= types, sorted(want - types)
    a = _schedule_run(model, q, 0)
    b = _schedule_run(model, q, 1)
    c = _schedule_run(model, q, 2)
    assert np.isfinite(a[0]).all() and np.abs(a[0] - q).max() > 0
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    assert np.array_equal(a[0], c[0]) and np.array_equal(a[1], c[1])
