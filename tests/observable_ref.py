"""Independent restatement of the observable sampling rule and the device corruptors (b2s_obs_modifiers, include/b2s.h), for the tests.

Timers: the reference's Observable.reset / Observable.update with delay 0 (utils/observables.py:214-259), called by MujocoEnv.reset
with force=True and after every substep's step2 (environments/base.py:418-427, 494-505).  Python floats, as the reference runs them.
Noise: numpy restatement of obs_corrupt (csrc/b2s_ctrl.cuh) with tests.dynamics_override_host.philox4x32_10; bit-exact except
for log / cos / sqrt, which may differ from the device's by an ulp."""
import math

import numpy as np

from robosuite_b200.engine import CORRUPT_GAUSSIAN, CORRUPT_NONE, CORRUPT_UNIFORM, B2SError
from tests.dynamics_override_host import philox4x32_10


def obs_update(t, sampled, period, dt, force=False):
    """one Observable.update: (t, sampled) -> (t, sampled, took a sample)"""
    t += dt
    sample = False
    if force or (not sampled and period >= t):
        sample, sampled = True, True
    if t >= period:
        if not sampled:
            sample = True
        sampled = False
        t %= period
    return t, sampled, sample


def obs_reset(period, dt):
    """Observable.reset + the forced update of MujocoEnv.reset: (t, sampled)"""
    t, sampled, _ = obs_update(0.0, False, period, dt, force=True)
    return t, sampled


def sample_substeps(rate, dt, nsub, nsteps):
    """for each of `nsteps` control steps after a reset, the substeps (1-based) after which the observable samples"""
    period = 1.0 / rate
    t, sampled = obs_reset(period, dt)
    out = []
    for _ in range(nsteps):
        hits = []
        for sub in range(1, nsub + 1):
            t, sampled, s = obs_update(t, sampled, period, dt)
            if s:
                hits.append(sub)
        out.append(hits)
    return out


def _u53(w0, w1):
    return (((w0.astype(np.uint64) >> np.uint64(5)) << np.uint64(26)) | (w1.astype(np.uint64) >> np.uint64(6))).astype(np.float64) * 2.0 ** -53


def noise_uniforms(seed, env, count, rows):
    """(u1, u2) of rows `rows` of sample `count` of an environment: Philox counter (env, count, row, 0), key = seed"""
    rows = np.asarray(rows, dtype=np.uint64)
    ctr = np.zeros((len(rows), 4), dtype=np.uint64)
    ctr[:, 0], ctr[:, 1], ctr[:, 2] = int(env), int(count), rows
    x = philox4x32_10(ctr, (int(seed) & 0xFFFFFFFF, (int(seed) >> 32) & 0xFFFFFFFF))
    return _u53(x[:, 0], x[:, 1]), _u53(x[:, 2], x[:, 3])


def corrupt(values, mod, seed, env, count, rows):
    """the corrupted values of rows `rows` (float64 array `values`) of one observable's sample; mod = (period, kind, p0, p1, lo, hi)"""
    _, kind, p0, p1, lo, hi = mod
    v = np.asarray(values, dtype=np.float64)
    if kind == CORRUPT_NONE:
        return v
    u1, u2 = noise_uniforms(seed, env, count, rows)
    if kind == CORRUPT_GAUSSIAN:
        d = p0 + p1 * (np.sqrt(-2.0 * np.log(1.0 - u1)) * np.cos(2.0 * np.pi * u2))
    else:
        d = p0 + (p1 - p0) * u1
    return np.minimum(np.maximum(v + d, lo), hi)


def quat2mat(q_xyzw):
    """the reference's quat2mat (utils/transform_utils.py) in fp64: the quaternion is normalised (q *= sqrt(2 / n)), the identity when
    n < 4 eps - what a lagged `{obj}_to_robot0_eef_quat` builds from a corrupted `{obj}_quat` cache"""
    q = np.asarray(q_xyzw, dtype=np.float64)[[3, 0, 1, 2]].copy()
    n = float(np.dot(q, q))
    if n < np.finfo(float).eps * 4.0:
        return np.identity(3)
    q *= math.sqrt(2.0 / n)
    q2 = np.outer(q, q)
    return np.array([[1.0 - q2[2, 2] - q2[3, 3], q2[1, 2] - q2[3, 0], q2[1, 3] + q2[2, 0]],
                     [q2[1, 2] + q2[3, 0], 1.0 - q2[1, 1] - q2[3, 3], q2[2, 3] - q2[1, 0]],
                     [q2[1, 3] - q2[2, 0], q2[2, 3] + q2[1, 0], 1.0 - q2[1, 1] - q2[2, 2]]])


def check_modifiers(obs_dim, row_obs, mods):
    """the argument checks of b2s_obs_modifiers (B2SError, as the library's return code surfaces)"""
    if len(mods) > 32:
        raise B2SError("b2s_obs_modifiers: nobs must be in [0, 32]")
    for o, (period, kind, p0, p1, lo, hi) in enumerate(mods):
        if not (period > 0 and math.isfinite(period)):
            raise B2SError("observable %d: the period must be finite and > 0" % o)
        if kind not in (CORRUPT_NONE, CORRUPT_GAUSSIAN, CORRUPT_UNIFORM):
            raise B2SError("observable %d: unknown corruptor" % o)
        if kind != CORRUPT_NONE:
            if not (math.isfinite(p0) and math.isfinite(p1)):
                raise B2SError("observable %d: noise parameters must be finite" % o)
            if kind == CORRUPT_GAUSSIAN and p1 < 0:
                raise B2SError("observable %d: std < 0" % o)
            if kind == CORRUPT_UNIFORM and p1 < p0:
                raise B2SError("observable %d: max_noise < min_noise" % o)
            if not lo <= hi:
                raise B2SError("observable %d: low > high" % o)
    if mods:
        r = np.asarray(row_obs)
        if len(r) < obs_dim or np.any(r[:obs_dim] < 0) or np.any(r[:obs_dim] >= len(mods)):
            raise B2SError("b2s_obs_modifiers: a row is mapped out of range")
