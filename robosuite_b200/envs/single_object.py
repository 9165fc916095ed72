"""single_object_mode of the multi-object tasks (PickPlace, NutAssembly), shared by both task classes.

Recalled from robosuite v1.5.2 (environments/manipulation/pick_place.py, nut_assembly.py; no reference checkout was at hand to pin
line numbers):
  mode 0  every object is in play (the default);
  mode 1  every reset draws one object uniformly (`random.choice`), parks the others (`clear_objects`: qpos (10, 10, 10, 1, 0, 0, 0))
          and switches the observables of the drawn object on and of the others off; the index is an observable (`obj_id` /
          `nut_id`) at the end of the `object` modality;
  mode 2  one fixed object (`object_type` / `nut_type`); the others are parked at every reset.
Every object stays in the model and is simulated (a parked object falls onto the floor plane and rests there).  Placements are drawn
as in mode 0, so the active object's placement is still rejected against the objects placed before it.  Success: at least one
object placed (modes 1, 2); the staged rewards run over every object not yet placed, parked ones included.

Mode 1 here: the draw comes from `env.rng` on the device (the reference uses Python's `random`).  The batch shares one observation
table, so the object observables read the environment's object through the device's selection (BatchedSim.obs_objects, ops
OB_SEL_*); they are keyed `{key}_to_robot0_eef_pos`, `{key}_to_robot0_eef_quat`, `{key}_pos`, `{key}_quat` with key "obj" / "nut"
where the reference names them after the drawn object (a name that differs between the environments of a batch).  The flattened
rows are the reference's."""
from .base import OB_SEL_BODY_POS, OB_SEL_BODY_QUAT_XYZW, OB_SEL_INDEX

PARKED_QPOS = (10.0, 10.0, 10.0, 1.0, 0.0, 0.0, 0.0)  # environments/base.py clear_objects


def parse_mode(mode, type_name, type_to_id, arg):
    """(single_object_mode, fixed object index or None) from the constructor's arguments, with the reference's checks"""
    if mode not in (0, 1, 2):
        raise ValueError("invalid @single_object_mode argument {!r} - choose one of [0, 1, 2]".format(mode))
    msg = "invalid @{} argument - choose one of {}".format(arg, list(type_to_id.keys()))
    if type_name is not None and type_name not in type_to_id:
        raise ValueError(msg)
    if mode == 2 and type_name is None:
        raise ValueError(msg)
    return mode, (None if type_name is None else type_to_id[type_name])


def reject_fixed(kwargs, *names):
    """the registered single-object variants fix mode and object; the reference asserts "invalid set of arguments" """
    if any(n in kwargs for n in names):
        raise ValueError("invalid set of arguments: {} fixes {}".format("this task", " and ".join(names)))


class SingleObjectMixin:
    """Object selection, parking and the selected-object observables.  The task class provides `single_object_mode`,
    `_fixed_object` (index or None), `_object_names` (the objects in index order), `obj_body_id` and `obj_qadr`."""

    single_object_mode = 0
    _fixed_object = None
    _sel = None  # the engine's obj_sel [N] int32 (mode 1)

    @property
    def object_id(self):
        """the object in play: mode 1 the per-environment selection (the engine's obj_sel, [N] int32 on the device, carried by its
        snapshots); mode 2 the fixed index; mode 0 None"""
        if self.single_object_mode == 1:
            return self._sel
        return self._fixed_object if self.single_object_mode == 2 else None

    def _setup_selection(self):
        if self.single_object_mode == 1:
            self._sel = self.sim.obs_objects([self.obj_body_id[n] for n in self._object_names])

    def _add_selected_object_obs(self, ob, key, id_name):
        ob.add_rel_pose(key, self.eef_site_id, self.eef_body_id, "object")
        ob.add(key + "_pos", "object", [(OB_SEL_BODY_POS, 0, k) for k in range(3)])
        ob.add(key + "_quat", "object", [(OB_SEL_BODY_QUAT_XYZW, 0, k) for k in range(4)])
        ob.add(id_name, "object", [(OB_SEL_INDEX, 0, 0)])

    def _park_objects(self, q):
        """after the placements (all objects, mode 0's draws): mode 2 parks all but the fixed object; mode 1 draws one object per
        environment (one more draw from env.rng), parks the others and keeps the draw in `_sel_draw` [N] for _randomize_model, which
        BatchedMujocoEnv.reset calls next with the reset's mask"""
        import torch

        if self.single_object_mode == 0:
            return
        n, k = q.shape[0], len(self._object_names)
        if self.single_object_mode == 1:
            self._sel_draw = torch.randint(0, k, (n,), generator=self.rng, device=self.device, dtype=torch.int64)
            keep = [self._sel_draw == i for i in range(k)]
        else:
            keep = [None] * k
        park = self._dev_const("parked_qpos", PARKED_QPOS)
        for i, name in enumerate(self._object_names):
            a = self.obj_qadr[name]
            if self.single_object_mode == 2:
                if i != self._fixed_object:
                    q[:, a:a + 7] = park
            else:
                q[:, a:a + 7] = torch.where(keep[i][:, None], q[:, a:a + 7], park)

    def _randomize_model(self, mask):
        import torch

        super()._randomize_model(mask)
        if self.single_object_mode == 1:  # the masked environments take this reset's draw, on the device
            draw = self._sel_draw.to(torch.int32)
            self._sel.copy_(draw if mask is None else torch.where(mask, draw, self._sel))
