"""Object placement samplers with the reference's names, arguments and defaults (robosuite/utils/placement_samplers.py), for
`make(task, placement_initializer=...)`.

Recalled from robosuite v1.5 (no reference checkout was at hand to check them against): the constructor signatures and defaults
below, `sample()`'s rules (base offset from `reference_pos` or a `reference` object / vector, x and y = numpy's uniform over the
ranges shrunk by the object's horizontal radius when `ensure_object_boundary_in_range`, z = z_offset + base z minus the bottom offset
when `on_top`, the overlap rule of `ensure_valid_placement`, up to 5000 tries per object, the rotation forms of `_sample_quat`),
`SequentialCompositeSampler.hide`'s ranges and how the tasks' `_load_model` hands their objects to a given sampler (`reset()`, then
`add_objects`).

Nothing is sampled on the host: a task lowers its sampler once, at construction, into a flat per-object program
(`lower`), and every reset places the objects of the environments being reset on the device in one launch
(BatchedSim.place_objects, include/b2s.h b2s_place_objects).  Objects are given by the task's object names ("cube"; "cubeA",
"cubeB"; "SquareNut", "RoundNut"; "Door"), because the task's MujocoObject instances do not exist before the environment does."""
import math
import numbers
from collections import OrderedDict

from .errors import RandomizationError  # noqa: F401  (the reference's module exports it too)

MAX_ROTATION_RANGES = 8  # (min, max) pairs a list-of-ranges rotation may hold (b2s_place: B2S_PLACE_MAXROT)


def _finite(v, what):
    if isinstance(v, bool) or not isinstance(v, numbers.Real) or not math.isfinite(float(v)):
        raise ValueError("{} must be a finite number, got {!r}".format(what, v))
    return float(v)


def _finite_vec(v, n, what):
    try:
        vals = list(v)
    except TypeError:
        raise ValueError("{} must hold {} finite numbers, got {!r}".format(what, n, v))
    if len(vals) != n:
        raise ValueError("{} must hold {} finite numbers, got {!r}".format(what, n, v))
    return tuple(_finite(x, what) for x in vals)


def _names(mujoco_objects):
    objs = [mujoco_objects] if isinstance(mujoco_objects, str) else list(mujoco_objects)
    for o in objs:
        if not isinstance(o, str):
            raise TypeError("objects are given by the task's object names (str), got {!r}".format(o))
    return objs


class ObjectPositionSampler:
    """Base class of the samplers (placement_samplers.py ObjectPositionSampler)."""

    def __init__(self, name, mujoco_objects=None, ensure_object_boundary_in_range=True, ensure_valid_placement=True,
                 reference_pos=(0, 0, 0), z_offset=0.0):
        self.name = name
        self.mujoco_objects = [] if mujoco_objects is None else _names(mujoco_objects)
        self.ensure_object_boundary_in_range = bool(ensure_object_boundary_in_range)
        self.ensure_valid_placement = bool(ensure_valid_placement)
        self.reference_pos = _finite_vec(reference_pos, 3, "reference_pos")
        self.z_offset = _finite(z_offset, "z_offset")

    def add_objects(self, mujoco_objects):
        for obj in _names(mujoco_objects):
            if obj in self.mujoco_objects:
                raise ValueError("Object '{}' already in sampler!".format(obj))
            self.mujoco_objects.append(obj)

    def reset(self):
        """Removes all objects from this sampler."""
        self.mujoco_objects = []

    def sample(self, fixtures=None, reference=None, on_top=True):
        raise NotImplementedError("placements are drawn on the device at every reset of the environment the sampler was given to "
                                  "(make(..., placement_initializer=sampler)); read them from env.sim.qpos or env.door_pose")


class UniformRandomSampler(ObjectPositionSampler):
    """x, y uniform in x_range / y_range around the base offset, rotation per `rotation` about `rotation_axis`:
    None = U[0, 2 pi), a number = that angle, a (lo, hi) pair = U[min, max], a list of pairs = one pair drawn uniformly, then
    uniform in it (at most 8 pairs here)."""

    def __init__(self, name, mujoco_objects=None, x_range=(0, 0), y_range=(0, 0), rotation=None, rotation_axis="z",
                 ensure_object_boundary_in_range=True, ensure_valid_placement=True, reference_pos=(0, 0, 0), z_offset=0.0):
        self.x_range = _finite_vec(x_range, 2, "x_range")
        self.y_range = _finite_vec(y_range, 2, "y_range")
        self.rotation = rotation
        self._rotation_ranges = self._lower_rotation(rotation)
        if rotation_axis not in ("x", "y", "z"):
            raise ValueError("Invalid rotation axis specified. Must be 'x', 'y', or 'z'. Got: {}".format(rotation_axis))
        self.rotation_axis = rotation_axis
        super().__init__(name, mujoco_objects=mujoco_objects, ensure_object_boundary_in_range=ensure_object_boundary_in_range,
                         ensure_valid_placement=ensure_valid_placement, reference_pos=reference_pos, z_offset=z_offset)

    @staticmethod
    def _lower_rotation(rotation):
        """the rotation as (min, max) pairs, one drawn uniformly: U[0, 2 pi) = [(0, 2 pi)], an angle a = [(a, a)]"""
        if rotation is None:
            return [(0.0, 2 * math.pi)]
        if isinstance(rotation, numbers.Real) and not isinstance(rotation, bool):
            a = _finite(rotation, "rotation")
            return [(a, a)]
        items = list(rotation)
        if items and not isinstance(items[0], numbers.Real):  # a list of ranges (random.choice of one)
            if not 1 <= len(items) <= MAX_ROTATION_RANGES:
                raise ValueError("a list of rotation ranges holds 1 to {} ranges, got {}".format(MAX_ROTATION_RANGES, len(items)))
            pairs = [list(r) for r in items]
        else:
            pairs = [items]
        out = []
        for p in pairs:
            if len(p) < 1:
                raise ValueError("a rotation range needs at least one angle, got {!r}".format(rotation))
            vals = [_finite(a, "rotation") for a in p]
            out.append((min(vals), max(vals)))  # np.random.uniform(high=max(rotation), low=min(rotation))
        return out


class SequentialCompositeSampler(ObjectPositionSampler):
    """Runs its samplers in order; each one sees every placement made before it.  `sample_args` of a sampler may set `reference`
    (the name of an object placed earlier, or a 3-vector) and `on_top`."""

    def __init__(self, name):
        self.samplers = OrderedDict()
        self.sample_args = OrderedDict()
        super().__init__(name=name)

    def append_sampler(self, sampler, sample_args=None):
        for obj in sampler.mujoco_objects:
            if obj in self.mujoco_objects:
                raise ValueError("Object '{}' already has sampler associated with it!".format(obj))
        if sample_args is not None:
            unknown = set(sample_args) - {"reference", "on_top"}
            if unknown:
                raise ValueError("sample_args may set 'reference' and 'on_top', got {}".format(sorted(unknown)))
            ref = sample_args.get("reference")
            if ref is not None and not isinstance(ref, str):
                _finite_vec(ref, 3, "reference")
        self.samplers[sampler.name] = sampler
        self.sample_args[sampler.name] = sample_args
        self.mujoco_objects += sampler.mujoco_objects

    def hide(self, mujoco_objects):
        """parks objects far away: x, y in [-10, -20], rotation [0, 0] about z, z_offset 10, no boundary or validity checks"""
        sampler = UniformRandomSampler(name="HideSampler", mujoco_objects=mujoco_objects, x_range=[-10, -20], y_range=[-10, -20],
                                       rotation=[0, 0], rotation_axis="z", z_offset=10, ensure_object_boundary_in_range=False,
                                       ensure_valid_placement=False)
        self.append_sampler(sampler=sampler)

    def add_objects_to_sampler(self, sampler_name, mujoco_objects):
        self.add_objects(mujoco_objects)
        self.samplers[sampler_name].add_objects(mujoco_objects)

    def reset(self):
        super().reset()
        for sampler in self.samplers.values():
            sampler.reset()


_AXIS = {"x": 0, "y": 1, "z": 2}


def lower(sampler, objects):
    """The flat program of `sampler` over the task's `objects` (name -> dict(radius, bottom, top, qpos_adr, body): horizontal
    radius, bottom and top offsets along z, and the target, a free joint's qpos address or a world-welded body with a pose override,
    -1 for the other): one entry per object in placement order, the fields of BatchedSim.place_config.  Returns (names, entries).
    ValueError: an unknown object, an object placed twice, a task object no sampler places, a `reference` name not placed earlier."""
    names, entries = [], []

    def run(s, reference, on_top):
        if isinstance(s, SequentialCompositeSampler):
            for key, sub in s.samplers.items():
                args = dict(s.sample_args[key] or {})
                run(sub, args.get("reference", reference), args.get("on_top", on_top))
            return
        if not isinstance(s, UniformRandomSampler):
            raise NotImplementedError("placement on the device implements UniformRandomSampler and SequentialCompositeSampler, got {}"
                                      .format(type(s).__name__))
        for name in s.mujoco_objects:
            if name not in objects:
                raise ValueError("sampler '{}': unknown object '{}' (this task's objects: {})".format(s.name, name, list(objects)))
            if name in names:
                raise ValueError("Object '{}' has already been sampled!".format(name))
            meta = objects[name]
            x_min, x_max = s.x_range
            y_min, y_max = s.y_range
            if s.ensure_object_boundary_in_range:
                r = float(meta["radius"])
                x_min, x_max, y_min, y_max = x_min + r, x_max - r, y_min + r, y_max - r
            ref, ref_dz, base = -1, 0.0, s.reference_pos
            if isinstance(reference, str):
                if reference not in names:
                    raise ValueError("sampler '{}': reference object '{}' is not placed before '{}'".format(s.name, reference, name))
                ref, base = names.index(reference), (0.0, 0.0, 0.0)
                ref_dz = float(objects[reference]["top"]) if on_top else 0.0
            elif reference is not None:
                base = _finite_vec(reference, 3, "reference")
            entries.append(dict(qpos_adr=int(meta.get("qpos_adr", -1)), body=int(meta.get("body", -1)), ref=ref,
                                ensure_valid=s.ensure_valid_placement, axis=_AXIS[s.rotation_axis], x_min=x_min, x_max=x_max,
                                y_min=y_min, y_max=y_max, base=tuple(base), ref_dz=ref_dz, z_offset=s.z_offset,
                                bottom_dz=float(meta["bottom"]) if on_top else 0.0, radius=float(meta["radius"]),
                                bottom=float(meta["bottom"]), top=float(meta["top"]), rot=list(s._rotation_ranges)))
            names.append(name)

    run(sampler, None, True)
    missing = [n for n in objects if n not in names]
    if missing:
        raise ValueError("no sampler of '{}' places the task's object(s) {}".format(sampler.name, missing))
    return names, entries
