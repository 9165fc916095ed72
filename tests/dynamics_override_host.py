"""Host side of the per-environment joint and contact fields and of the device perturbation, for the tests:
- dynamics_override_model: a copy of a model with per-object values of all nine per-environment fields and the compiler's
  set-constants step re-run (the oracle of an environment is built from it);
- dynamics_invalid: warn bit 128 of the set-constants pass;
- philox4x32_10 / perturb_values: a numpy restatement of b2s_perturb_model (include/b2s.h) that reproduces its draws bit for bit."""
import copy

import numpy as np

from robosuite_b200.engine import DOF_FIELDS, GEOM_CONTACT_FIELDS, PERTURB_SCALE, normalize_perturb_spec
from tests.model_override_host import FIELDS, invalid, override_model

ALL_FIELDS = FIELDS + GEOM_CONTACT_FIELDS + DOF_FIELDS


def dynamics_override_model(model, **vals):
    """`vals`: field -> {object id: value}; the dof fields take the whole vector under id -1"""
    m = copy.deepcopy(model)
    for f in GEOM_CONTACT_FIELDS:
        for g, v in (vals.get(f) or {}).items():
            getattr(m, f)[g] = np.asarray(v, dtype=np.float64)
    for f in DOF_FIELDS:
        for _, v in (vals.get(f) or {}).items():
            setattr(m, f, np.asarray(v, dtype=np.float64).copy())
    return override_model(m, **{f: vals.get(f) for f in FIELDS})


def dynamics_invalid(model, **vals):
    bad = invalid(model, **{f: vals.get(f) for f in FIELDS})
    for f in GEOM_CONTACT_FIELDS:
        bad |= any(not np.all(np.isfinite(np.asarray(v, dtype=np.float64))) for v in (vals.get(f) or {}).values())
    for f in DOF_FIELDS:
        for v in (vals.get(f) or {}).values():
            v = np.asarray(v, dtype=np.float64)
            bad |= not bool(np.all(np.isfinite(v)) and np.all(v >= 0))
    return bool(bad)


_MASK = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """Philox4x32-10 (Salmon et al., SC'11) on [..., 4] uint32 counters with a (k0, k1) key -> [..., 4] uint32"""
    c = [np.asarray(ctr, dtype=np.uint64)[..., i] for i in range(4)]
    k0, k1 = np.uint64(key[0]), np.uint64(key[1])
    for r in range(10):
        if r:
            k0, k1 = (k0 + np.uint64(0x9E3779B9)) & _MASK, (k1 + np.uint64(0xBB67AE85)) & _MASK
        p0, p1 = np.uint64(0xD2511F53) * c[0], np.uint64(0xCD9E8D57) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & _MASK, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & _MASK]
    return np.stack(c, axis=-1).astype(np.uint32)


def model_values(model, field, obj_id):
    """the model's value(s) an entry perturbs around, as a 1-d float64 array"""
    v = np.asarray(getattr(model, field), dtype=np.float64)
    if field in DOF_FIELDS:
        return v.copy() if obj_id < 0 else v[obj_id:obj_id + 1].copy()
    return np.atleast_1d(v[obj_id]).astype(np.float64)


def perturb_values(model, spec, envs, seed, counter):
    """values b2s_perturb_model writes: {entry index: float64 [len(envs), ncomp]} for environments `envs`"""
    envs = np.asarray(envs, dtype=np.uint64)
    key = (int(seed) & 0xFFFFFFFF, (int(seed) >> 32) & 0xFFFFFFFF)
    out = {}
    for k, (field, oid, mode, amp, one) in enumerate(normalize_perturb_spec(spec)):
        base = model_values(model, field, oid)
        comp = np.zeros(len(base), dtype=np.uint64) if one else np.arange(len(base), dtype=np.uint64)
        ctr = np.zeros((len(envs), len(base), 4), dtype=np.uint64)
        ctr[..., 0] = envs[:, None]
        ctr[..., 1] = int(counter)
        ctr[..., 2] = k
        ctr[..., 3] = comp[None, :]
        x = philox4x32_10(ctr, key).astype(np.uint64)
        u = (((x[..., 0] >> np.uint64(5)) << np.uint64(26)) | (x[..., 1] >> np.uint64(6))).astype(np.float64) * 2.0 ** -53
        d = amp * (2.0 * u - 1.0)
        out[k] = base[None, :] * (1.0 + d) if mode == PERTURB_SCALE else np.maximum(0.0, base[None, :] + d)
    return out
