"""Contact queries of the batched environments: `check_contact`, `get_contacts` and `_check_grasp` over the contacts of the last
substep of the last step, one answer per environment, computed with torch on the device (no host synchronisation).

Recalled from robosuite v1.5.2 (utils/sim_utils.py:8-67 check_contact / get_contacts, environments/manipulation/manipulation_env.py
:331-376 _check_grasp; no reference checkout was at hand to re-read them).  Each reads sim.data.contact[:ncon] after env.step:
  check_contact(geoms_1, geoms_2=None)  True when some contact (g1, g2) has (g1 in A and (B is None or g2 in B)) or
                                        (g2 in A and (B is None or g1 in B)), A = geoms_1, B = geoms_2;
  get_contacts(model)                   the set of geoms in contact with the model: for each contact with exactly one geom in
                                        model.contact_geoms, the other geom;
  _check_grasp(gripper, object_geoms)   True when every fingerpad group of the gripper (left, right) is in contact with the object
                                        geoms (check_contact(group, object_geoms) for each group).
The reference takes geom names and MujocoModel objects; here a geom argument is a name, a list of names, an id, or a list / tensor
of ids, and `contact_geoms(prefix)` stands in for RobotModel.contact_geoms.  get_contacts returns a [N, ngeom] bool mask (the batched
form of the name set) and _check_grasp takes the object first, its gripper defaulting to the environment's fingerpad groups.

The queries read the arrays BatchedSim.set_contact_export fills on the last substep of every step in every schedule; an environment
made without `contact_queries=True` has no such arrays to read, and the queries raise instead of answering from stale contacts.
reset() writes the reset environments' contacts (its forward pass); set_env_state / clone_envs run no physics, so until the next
step the queries answer from the contacts the environments had before."""
import numpy as np


class ContactQueries:
    """mixed into BatchedMujocoEnv; needs `sim`, `model`, `device` and `_contact_queries`"""

    def _contacts_or_raise(self):
        if not getattr(self, "_contact_queries", False):
            raise RuntimeError("contact queries need the contact export: create the environment with "
                               "make(..., contact_queries=True)")
        return self.sim.contacts()

    def contact_geoms(self, prefix):
        """ids of the colliding geoms (those in at least one collision pair) whose names start with `prefix`, e.g. "robot0_" or
        "gripper0_" (RobotModel.contact_geoms / GripperModel.contact_geoms of the reference)"""
        m = self.model
        colliding = {int(g) for p in m.pair_geom for g in p}
        return [g for g, n in enumerate(m.names["geom"]) if g in colliding and n and n.startswith(prefix)]

    def _geom_ids(self, geoms):
        """host list of geom ids of a name, an id, or a list / array / host tensor of names and ids; ValueError for an unknown name
        or an id out of range"""
        import torch

        if isinstance(geoms, (str, int, np.integer)):
            geoms = [geoms]
        elif torch.is_tensor(geoms):
            geoms = geoms.reshape(-1).tolist()
        names, ng = self.model.names["geom"], int(self.model.ngeom)
        ids = []
        for g in geoms:
            if isinstance(g, str):
                if g not in names:
                    raise ValueError("unknown geom name {!r}".format(g))
                ids.append(names.index(g))
            else:
                k = int(g)
                if not 0 <= k < ng:
                    raise ValueError("geom id {} out of range [0, {})".format(k, ng))
                ids.append(k)
        return ids

    def _geom_mask(self, geoms):
        """bool [ngeom + 1] device mask of a geom argument (slot ngeom: the -1 of the unused contact rows, never set).  A tensor of
        ids already on the device is used as it is, without a range check (that would synchronise): ids outside [0, ngeom) match
        nothing.  Masks of host arguments are uploaded once per geom set."""
        import torch

        ng = int(self.model.ngeom)
        if torch.is_tensor(geoms) and geoms.device.type == "cuda":
            ids = geoms.reshape(-1).to(device=self.device, dtype=torch.long)
            mask = torch.zeros(ng + 1, dtype=torch.bool, device=self.device)
            mask[torch.where((ids >= 0) & (ids < ng), ids, ng)] = True
            mask[ng] = False
            return mask
        ids = tuple(sorted(set(self._geom_ids(geoms))))
        cache = self.__dict__.setdefault("_geom_masks", {})
        if ids not in cache:
            mask = np.zeros(ng + 1, dtype=bool)
            mask[list(ids)] = True
            cache[ids] = torch.as_tensor(mask, device=self.device)
        return cache[ids]

    def _contact_pairs(self):
        """(g1, g2) long [N, maxcon] with the unused rows (and any row at or beyond ncon) mapped to the sentinel slot ngeom"""
        import torch

        c = self._contacts_or_raise()
        ng = int(self.model.ngeom)
        g = c["geom"].long()
        live = torch.arange(g.shape[1], device=g.device)[None, :] < c["ncon"].long()[:, None]
        g = torch.where(live[..., None] & (g >= 0), g, ng)
        return g[..., 0], g[..., 1]

    def check_contact(self, geoms_1, geoms_2=None):
        """bool [N]: some contact of the last substep is between geoms_1 and geoms_2 (any geom when geoms_2 is None)"""
        g1, g2 = self._contact_pairs()
        a = self._geom_mask(geoms_1)
        a1, a2 = a[g1], a[g2]
        if geoms_2 is None:
            hit = a1 | a2
        else:
            b = self._geom_mask(geoms_2)
            hit = (a1 & b[g2]) | (a2 & b[g1])
        return hit.any(dim=1)

    def get_contacts(self, geoms):
        """bool [N, ngeom]: the geoms in contact with `geoms` - the other geom of every contact with exactly one geom in the set"""
        import torch

        g1, g2 = self._contact_pairs()
        s = self._geom_mask(geoms)
        s1, s2 = s[g1], s[g2]
        ng = int(self.model.ngeom)
        other = torch.where(s1 & ~s2, g2, torch.where(s2 & ~s1, g1, ng))
        out = torch.zeros((other.shape[0], ng + 1), dtype=torch.bool, device=other.device)
        out.scatter_(1, other, True)
        return out[:, :ng]

    def _check_grasp(self, object_geoms, gripper=None):
        """bool [N]: every gripper group touches the object geoms.  gripper None: the environment's left and right fingerpad groups;
        a name or id: one group of that geom; a list: one group per element (a name, an id, or a list of them)"""
        if gripper is None:
            groups = list(self._fingerpad_geoms())
        elif isinstance(gripper, (str, int, np.integer)):
            groups = [[gripper]]
        else:
            groups = [[g] if isinstance(g, (str, int, np.integer)) else g for g in gripper]
        import torch

        out = torch.ones(self.num_envs, dtype=torch.bool, device=self.device)
        for grp in groups:
            out &= self.check_contact(grp, object_geoms)
        return out
