"""Host restatements of object placement, for the tests:
- place_values: a numpy restatement of b2s_place_objects (include/b2s.h, csrc/b2s_place.cuh) that walks each object's tries in
  order with the same Philox4x32-10 draws (tests/dynamics_override_host.philox4x32_10) and the same fp64 operations, including the
  library's sin / cos sequence (sincos), so that it reproduces the device's q rows and pose overrides bit for bit;
- reference_sample: a literal transcription of the reference's UniformRandomSampler / SequentialCompositeSampler.sample loop
  (robosuite/utils/placement_samplers.py, recalled from robosuite v1.5), fed from a uniform stream instead of numpy's / Python's
  global generators."""
import math

import numpy as np

from tests.dynamics_override_host import philox4x32_10

TRIES = 5000
ROT_WORD = 0xFFFFFFFF


def _u53(a, b):
    a, b = np.asarray(a, dtype=np.uint64), np.asarray(b, dtype=np.uint64)
    return (((a >> np.uint64(5)) << np.uint64(26)) | (b >> np.uint64(6))).astype(np.float64) * 2.0 ** -53


def _draws(seed, counter, env, o, t):
    """(u for words 0-1, u for words 2-3) of counter (env, counter, o, t); t may be an array"""
    t = np.atleast_1d(np.asarray(t, dtype=np.uint64))
    ctr = np.zeros((len(t), 4), dtype=np.uint64)
    ctr[:, 0], ctr[:, 1], ctr[:, 2], ctr[:, 3] = env, counter, o, t
    w = philox4x32_10(ctr, (int(seed) & 0xFFFFFFFF, (int(seed) >> 32) & 0xFFFFFFFF)).astype(np.uint64)
    return _u53(w[:, 0], w[:, 1]), _u53(w[:, 2], w[:, 3])


_S = (-1.66666666666666324348e-01, 8.33333333332248946124e-03, -1.98412698298579493134e-04, 2.75573137070700676789e-06,
      -2.50507602534068634195e-08, 1.58969099521155010221e-10)
_C = (4.16666666666666019037e-02, -1.38888888888741095749e-03, 2.48015872894767294178e-05, -2.75573143513906633035e-07,
      2.08757232129817482790e-09, -1.13596475577881948265e-11)


def sincos(a):
    """place_sincos of csrc/b2s_place.cuh, operation for operation (numpy float64: every operation rounded once)"""
    a = np.float64(a)
    k = np.rint(a * np.float64(6.36619772367581382433e-01))
    r = (a - k * np.float64(1.57079632673412561417e+00)) - k * np.float64(6.07710050650619224932e-11)
    z = r * r
    ps = np.float64(_S[4]) + z * np.float64(_S[5])
    for c in (_S[3], _S[2], _S[1], _S[0]):
        ps = np.float64(c) + z * ps
    s = r + (z * r) * ps
    pc = np.float64(_C[4]) + z * np.float64(_C[5])
    for c in (_C[3], _C[2], _C[1], _C[0]):
        pc = np.float64(c) + z * pc
    hz = np.float64(0.5) * z
    w = np.float64(1.0) - hz
    c = w + (((np.float64(1.0) - w) - hz) + z * (z * pc))
    return {0: (s, c), 1: (c, -s), 2: (-s, -c), 3: (-c, s)}[int(k) & 3]


def quat_mat(q):
    w, x, y, z = (np.float64(v) for v in q)
    two = np.float64(2.0)
    return [((w * w + x * x) - y * y) - z * z, two * (x * y - w * z), two * (x * z + w * y),
            two * (x * y + w * z), ((w * w - x * x) + y * y) - z * z, two * (y * z - w * x),
            two * (x * z - w * y), two * (y * z + w * x), ((w * w - x * x) - y * y) + z * z]


def quat_mul(a, b):
    a0, a1, a2, a3 = (np.float64(v) for v in a)
    b0, b1, b2, b3 = (np.float64(v) for v in b)
    return [((a0 * b0 - a1 * b1) - a2 * b2) - a3 * b3, ((a0 * b1 + a1 * b0) + a2 * b3) - a3 * b2,
            ((a0 * b2 - a1 * b3) + a2 * b0) + a3 * b1, ((a0 * b3 + a1 * b2) - a2 * b1) + a3 * b0]


def compose(pos, quat, lp, lq):
    """placed pose * (lp, lq), as the kernel writes the override of a body welded to the placed one"""
    M = quat_mat(quat)
    p = [np.float64(pos[r]) + ((M[3 * r] * np.float64(lp[0]) + M[3 * r + 1] * np.float64(lp[1])) + M[3 * r + 2] * np.float64(lp[2]))
         for r in range(3)]
    return p, quat_mul(quat, lq)


def place_env(entries, seed, counter, env):
    """one environment: [(pos (3), quat (4), try index or -1 when none was valid)] per entry, walking the tries in order"""
    out = []
    for o, e in enumerate(entries):
        f = np.float64
        if e["ref"] >= 0:
            rp = out[e["ref"]][0]
            bx, by, bz = rp[0], rp[1], rp[2] + f(e["ref_dz"])
        else:
            bx, by, bz = (f(v) for v in e["base"])
        z = (f(e["z_offset"]) + bz) - f(e["bottom_dz"])
        ux, uy = _draws(seed, counter, env, o, np.arange(TRIES))
        wx, wy = f(e["x_max"]) - f(e["x_min"]), f(e["y_max"]) - f(e["y_min"])
        chosen = -1
        for t in range(TRIES):
            x = (f(e["x_min"]) + wx * ux[t]) + bx
            y = (f(e["y_min"]) + wy * uy[t]) + by
            ok = True
            if e["ensure_valid"]:
                for j in range(o):
                    (ox, oy, oz), q = out[j][0], entries[j]
                    dx, dy = x - ox, y - oy
                    if np.sqrt(dx * dx + dy * dy) <= f(q["radius"]) + f(e["radius"]) and z - oz <= f(q["top"]) - f(e["bottom"]):
                        ok = False
                        break
            if ok:
                chosen = t
                break
        if chosen < 0:  # the environment keeps the last try
            t = TRIES - 1
            x, y = (f(e["x_min"]) + wx * ux[t]) + bx, (f(e["y_min"]) + wy * uy[t]) + by
        uc, ua = (v[0] for v in _draws(seed, counter, env, o, ROT_WORD))
        rot = e["rot"]
        c = min(int(np.floor(uc * f(len(rot)))), len(rot) - 1) if len(rot) > 1 else 0
        lo, hi = f(rot[c][0]), f(rot[c][1])
        ang = lo + (hi - lo) * ua
        s, co = sincos(ang * f(0.5))
        q = [co, 0.0, 0.0, 0.0]
        q[1 + int(e["axis"])] = s
        out.append(([x, y, z], [np.float64(v) for v in q], chosen))
    return out


def place_values(entries, envs, seed, counter, nq=None, qpos=None, ov_local=None):
    """b2s_place_objects for environments `envs`: {"pos": [n, k, 3], "quat": [n, k, 4], "tries": [n, k], "warn": [n] (1024 / 0)};
    with qpos (float64 [N, nq], modified in place) the free-joint entries are written into its rows; ov_local {entry index:
    [(lp, lq), ...]} gives "ov" {entry index: [[(pos, quat) per override] per env]} (override 0 = the placed pose itself)"""
    res = {"pos": [], "quat": [], "tries": [], "warn": [], "ov": {}}
    for env in envs:
        pl = place_env(entries, seed, counter, int(env))
        res["pos"].append([p for p, _, _ in pl])
        res["quat"].append([q for _, q, _ in pl])
        res["tries"].append([t for _, _, t in pl])
        res["warn"].append(1024 if any(t < 0 for _, _, t in pl) else 0)
        for o, e in enumerate(entries):
            if e["qpos_adr"] >= 0 and qpos is not None:
                a = int(e["qpos_adr"])
                qpos[int(env), a:a + 7] = np.array(pl[o][0] + pl[o][1], dtype=np.float64)
            if ov_local is not None and o in ov_local:
                poses = [(pl[o][0], pl[o][1])] + [compose(pl[o][0], pl[o][1], lp, lq) for lp, lq in ov_local[o]]
                res["ov"].setdefault(o, []).append(poses)
    for k in ("pos", "quat", "tries", "warn"):
        res[k] = np.asarray(res[k])
    return res


# ---- the reference's sample() loop, transcribed (fed from `rng`: uniform_xy / uniform_rot / choice, and start_object)
class _Obj:
    def __init__(self, name, meta):
        self.name = name
        self.horizontal_radius = meta["radius"]
        self.bottom_offset = np.array([0, 0, meta["bottom"]])
        self.top_offset = np.array([0, 0, meta["top"]])


def _uniform_sample(s, objects, rng, fixtures=None, reference=None, on_top=True):
    placed_objects = {} if fixtures is None else dict(fixtures)
    base_offset = np.array(s.reference_pos)
    if reference is not None:
        if isinstance(reference, str):
            assert reference in placed_objects, "Invalid reference received. Current options are: {}, requested: {}".format(
                placed_objects.keys(), reference)
            ref_pos, _, ref_obj = placed_objects[reference]
            base_offset = np.array(ref_pos)
            if on_top:
                base_offset += np.array((0, 0, ref_obj.top_offset[-1]))
        else:
            base_offset = np.array(reference)
            assert base_offset.shape[0] == 3
    for name in s.mujoco_objects:
        obj = _Obj(name, objects[name])
        assert obj.name not in placed_objects, "Object '{}' has already been sampled!".format(obj.name)
        rng.start_object()
        horizontal_radius = obj.horizontal_radius
        bottom_offset = obj.bottom_offset
        success = False
        for i in range(TRIES):
            lo, hi = s.x_range
            if s.ensure_object_boundary_in_range:
                lo += horizontal_radius
                hi -= horizontal_radius
            object_x = rng.uniform_xy(high=hi, low=lo) + base_offset[0]
            lo, hi = s.y_range
            if s.ensure_object_boundary_in_range:
                lo += horizontal_radius
                hi -= horizontal_radius
            object_y = rng.uniform_xy(high=hi, low=lo) + base_offset[1]
            object_z = s.z_offset + base_offset[2]
            if on_top:
                object_z -= bottom_offset[-1]
            location_valid = True
            if s.ensure_valid_placement:
                for (x, y, z), _, other_obj in placed_objects.values():
                    if (np.linalg.norm((object_x - x, object_y - y)) <= other_obj.horizontal_radius + horizontal_radius
                            and object_z - z <= other_obj.top_offset[-1] - bottom_offset[-1]):
                        location_valid = False
                        break
            if location_valid:
                quat = _sample_quat(s, rng)
                pos = (object_x, object_y, object_z)
                placed_objects[obj.name] = (pos, quat, obj)
                success = True
                break
        if not success:
            from robosuite_b200.errors import RandomizationError

            raise RandomizationError("Cannot place all objects ):")
    return placed_objects


def _sample_quat(s, rng):
    import collections.abc

    rotation = s.rotation
    if rotation is None:
        rot_angle = rng.uniform_rot(high=2 * np.pi, low=0)
    elif isinstance(rotation, collections.abc.Iterable):
        if isinstance(rotation[0], collections.abc.Iterable):
            rotation = rng.choice(rotation)
        rot_angle = rng.uniform_rot(high=max(rotation), low=min(rotation))
    else:
        rot_angle = rotation
    if s.rotation_axis == "x":
        return np.array([np.cos(rot_angle / 2), np.sin(rot_angle / 2), 0, 0])
    elif s.rotation_axis == "y":
        return np.array([np.cos(rot_angle / 2), 0, np.sin(rot_angle / 2), 0])
    return np.array([np.cos(rot_angle / 2), 0, 0, np.sin(rot_angle / 2)])


def reference_sample(sampler, objects, rng, fixtures=None, reference=None, on_top=True):
    """sampler.sample(fixtures, reference, on_top) of the reference, recursing through SequentialCompositeSampler"""
    from robosuite_b200.placement_samplers import SequentialCompositeSampler

    if not isinstance(sampler, SequentialCompositeSampler):
        return _uniform_sample(sampler, objects, rng, fixtures, reference, on_top)
    placed_objects = {} if fixtures is None else dict(fixtures)
    for sampler_, s_args in zip(sampler.samplers.values(), sampler.sample_args.values()):
        s_args = {} if s_args is None else dict(s_args)
        for arg_name, arg in zip(("reference", "on_top"), (reference, on_top)):
            if arg_name not in s_args:
                s_args[arg_name] = arg
        new_placements = reference_sample(sampler_, objects, rng, fixtures=placed_objects, **s_args)
        placed_objects.update(new_placements)
    return placed_objects


class PhiloxStream:
    """the uniforms of the device's draws for one environment, in the order the transcription asks for them: tries of object o
    give (u_x, u_y) in turn, its rotation the choice and the angle"""

    def __init__(self, seed, counter, env):
        self.seed, self.counter, self.env, self.o = seed, counter, env, -1

    def start_object(self):
        self.o += 1
        self.ux, self.uy = _draws(self.seed, self.counter, self.env, self.o, np.arange(TRIES))
        self.uc, self.ua = (v[0] for v in _draws(self.seed, self.counter, self.env, self.o, ROT_WORD))
        self.k = 0

    def uniform_xy(self, low, high):
        u = (self.ux if self.k % 2 == 0 else self.uy)[self.k // 2]
        self.k += 1
        return low + (high - low) * u  # numpy's uniform(low, high)

    def uniform_rot(self, low, high):
        return low + (high - low) * self.ua

    def choice(self, seq):
        return seq[min(int(math.floor(self.uc * len(seq))), len(seq) - 1)]
