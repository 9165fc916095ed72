"""Host model with per-object override values: the CPU counterpart of b2s_model_override + b2s_set_const for the tests (the
oracle of an environment is built from it, and the device's set-constants pass is compared with what the compiler derives)."""
import copy

import numpy as np

from robosuite_b200.mjcf import compiler

FIELDS = ("geom_size", "geom_friction", "body_mass", "body_inertia")


def override_model(model, geom_size=None, geom_friction=None, body_mass=None, body_inertia=None):
    """Copy of `model` with {object id: value} applied per field: bounding radius and box of every resized geom by the compiler's
    per-type rules, then the compiler's set-constants step (dof_invweight0, body_invweight0, stat_meaninertia)."""
    m = copy.deepcopy(model)
    for g, v in (geom_size or {}).items():
        m.geom_size[g] = np.asarray(v, dtype=np.float64)
        _, _, m.geom_rbound[g], m.geom_aabb[g] = compiler.primitive_geom_props(int(m.geom_type[g]), m.geom_size[g])
    for g, v in (geom_friction or {}).items():
        m.geom_friction[g] = np.asarray(v, dtype=np.float64)
    for b, v in (body_mass or {}).items():
        m.body_mass[b] = float(v)
    for b, v in (body_inertia or {}).items():
        m.body_inertia[b] = np.asarray(v, dtype=np.float64)
    compiler._set_const(m)
    return m


def invalid(model, geom_size=None, geom_friction=None, body_mass=None, body_inertia=None):
    """warn bit 128 of the set-constants pass: a non-finite or non-positive value (the size components the geom type uses), or
    principal moments that violate the triangle inequality"""
    def pos(v):
        v = np.asarray(v, dtype=np.float64)
        return bool(np.all(np.isfinite(v)) and np.all(v > 0))

    used = {compiler.GEOM_SPHERE: 1, compiler.GEOM_CAPSULE: 2, compiler.GEOM_CYLINDER: 2}
    bad = any(not pos(np.asarray(v)[:used.get(int(model.geom_type[g]), 3)]) for g, v in (geom_size or {}).items())
    bad |= any(not pos(v) for v in (geom_friction or {}).values()) or any(not pos(v) for v in (body_mass or {}).values())
    for v in (body_inertia or {}).values():
        a, b, c = (float(x) for x in v)
        bad |= not pos(v) or a + b < c or a + c < b or b + c < a
    return bad
