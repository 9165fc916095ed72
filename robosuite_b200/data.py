"""Batched `MjData` view (`BatchedSim.data`): the step-1 arrays of every environment with a leading [N] axis, and the getters the
reference's binding offers over them, computed on the device.

Recalled from robosuite v1.5.2 (utils/binding_utils.py, class MjData; no reference checkout was at hand to re-read it).  The binding
delegates the data attributes to mujoco.MjData (body_xpos / body_xquat / body_xmat are data.xpos / xquat / xmat) and adds, for
obj in body, site and geom, with `id = model.<obj>_name2id(name)`:
  get_<obj>_xpos(name)    <obj>_xpos[id]                        (body: xpos[id])
  get_<obj>_xmat(name)    <obj>_xmat[id].reshape((3, 3))        (body: xmat[id])
  get_body_xquat(name)    xquat[id]
  get_<obj>_jacp(name)    jacp [3, nv] from mj_jacBody / mj_jacSite / mj_jacGeom
  get_<obj>_jacr(name)    jacr [3, nv] likewise
  get_<obj>_xvelp(name)   np.dot(get_<obj>_jacp(name), qvel)
  get_<obj>_xvelr(name)   np.dot(get_<obj>_jacr(name), qvel)
and an unknown name raises ValueError.  Here every getter also takes an id, and returns [N, ...]: positions [N, 3], quaternions
[N, 4] (w, x, y, z), matrices [N, 3, 3], Jacobians [N, 3, nv] (the library's Jacobian kernels), velocities [N, 3].  qM is the
DENSE [N, nv, nv] matrix (MuJoCo stores it sparse; full_m() is mj_fullM's dense copy), qfrc_bias / qfrc_passive are [N, nv].

The arrays are written by forward / reset (the masked environments) and, after env_step / step, only while the handle's
step-1 export (set_step1_export, make(..., data_queries=True)) or its full export (set_export) is on.  A read on a handle with
both off raises instead of answering from the poses of an earlier forward.  Poses of non-colliding (visual) geoms are never
computed: asking for one raises ValueError.  After restore / clone_envs no physics runs, so the arrays keep the poses the
environments had before until the next step.

The step-2 half (recalled the same way: mujoco.MjData fields the reference's code reads after env.step, and mujoco.mj_contactForce):
qacc (state, always current), qfrc_actuator, actuator_force, qfrc_smooth, qacc_smooth, qfrc_constraint [N, nv] / [N, nu], nefc [N],
the constraint rows efc_type, efc_D, efc_R, efc_aref, efc_force [N, maxefc] and efc_J [N, maxefc, nv] kept at capacity (the first
nefc[e] rows of environment e are valid), and solver_niter [N].  They need the step-2 export (set_step2_export,
make(..., dynamics_queries=True)) or the full export.  contact_force() is mj_contactForce for elliptic cones: contact c's force
and torque in its own frame (normal first, then the tangential and the torsional / rolling components) are
efc_force[efc_address : efc_address + dim], zero-padded to 6; a contact without rows (efc_address -1: not penetrating, or
dropped by the row budget) has zero force.  It also needs the contact records (set_contact_export, or the full export)."""


class BatchedData:
    """The batched MjData of a BatchedSim (or a stand-in with the same surface: the named arrays as attributes, jac_site /
    jac_body / jac_geom, full_m, `model`, and the `full_export` / `step1_export` / `step2_export` / `contact_export` flags)."""

    def __init__(self, sim):
        self._sim = sim
        m = sim.model
        self._count = {"body": int(m.nbody), "site": int(m.nsite), "geom": int(m.ngeom)}
        self._colliding = {int(g) for p in m.pair_geom for g in p}

    # what each kind of read needs: the BatchedSim flag of its export (the full export also serves) and the error without either
    _NEEDS = {
        "step1": ("step1_export", "sim.data reads the step-1 arrays, which env_step / step write only with the step-1 export on: "
                  "create the environment with make(..., data_queries=True) or call BatchedSim.set_step1_export(True)"),
        "step2": ("step2_export", "sim.data reads the step-2 arrays, which env_step / step write only with the step-2 export on: "
                  "create the environment with make(..., dynamics_queries=True) or call BatchedSim.set_step2_export(True)"),
        "contacts": ("contact_export", "contact_force() also reads the contact records, which env_step / step write only with the "
                     "contact export on: create the environment with make(..., dynamics_queries=True) or call "
                     "BatchedSim.set_contact_export(True)"),
    }

    def _require(self, kind):
        flag, msg = self._NEEDS[kind]
        if not (self._sim.full_export or getattr(self._sim, flag)):
            raise RuntimeError(msg)

    def _array(self, name, kind):
        self._require(kind)
        return getattr(self._sim, name)

    def _id(self, kind, obj):
        """id of a body / site / geom given by name or id; ValueError for an unknown name, an id out of range, or a non-colliding geom"""
        names = self._sim.model.names[kind]
        if isinstance(obj, str):
            if obj not in names:
                raise ValueError('No "{}" with name {!r} exists'.format(kind, obj))
            i = names.index(obj)
        else:
            i = int(obj)
            if not 0 <= i < self._count[kind]:
                raise ValueError("{} id {} out of range [0, {})".format(kind, i, self._count[kind]))
        if kind == "geom" and i not in self._colliding:
            raise ValueError("geom {!r} (id {}) is not a colliding geom: the engine never computes the poses of non-colliding "
                             "(visual) geoms".format(names[i], i))
        return i

    # ---- the data attributes, [N, k, ...] device views
    body_xpos = property(lambda self: self._array("xpos", "step1"))
    body_xquat = property(lambda self: self._array("xquat", "step1"))
    body_xmat = property(lambda self: self._array("xmat", "step1"))
    site_xpos = property(lambda self: self._array("site_xpos", "step1"))
    site_xmat = property(lambda self: self._array("site_xmat", "step1"))
    geom_xpos = property(lambda self: self._array("geom_xpos", "step1"))
    geom_xmat = property(lambda self: self._array("geom_xmat", "step1"))
    qM = property(lambda self: self._array("qM", "step1"))
    cdof = property(lambda self: self._array("cdof", "step1"))
    qfrc_bias = property(lambda self: self._array("qfrc_bias", "step1"))
    qfrc_passive = property(lambda self: self._array("qfrc_passive", "step1"))

    # ---- the step-2 arrays, [N, ...] device views; the row arrays at capacity (nefc says how many rows are valid)
    qacc = property(lambda self: self._sim.qacc)  # state: written by every step
    qfrc_actuator = property(lambda self: self._array("qfrc_actuator", "step2"))
    actuator_force = property(lambda self: self._array("actuator_force", "step2"))
    qfrc_smooth = property(lambda self: self._array("qfrc_smooth", "step2"))
    qacc_smooth = property(lambda self: self._array("qacc_smooth", "step2"))
    qfrc_constraint = property(lambda self: self._array("qfrc_constraint", "step2"))
    nefc = property(lambda self: self._array("nefc", "step2"))
    efc_type = property(lambda self: self._array("efc_type", "step2"))
    efc_J = property(lambda self: self._array("efc_J", "step2"))
    efc_D = property(lambda self: self._array("efc_D", "step2"))
    efc_R = property(lambda self: self._array("efc_R", "step2"))
    efc_aref = property(lambda self: self._array("efc_aref", "step2"))
    efc_force = property(lambda self: self._array("efc_force", "step2"))
    solver_niter = property(lambda self: self._array("solver_niter", "step2"))

    def contact_force(self, contact=None):
        """mj_contactForce of every contact slot, [N, maxcon, 6], or of slot `contact` (an int), [N, 6]: force and torque in the
        contact's frame (contact_frame), zeros for a contact without constraint rows and for slots at or beyond ncon.  Elliptic
        cones only (a pyramidal cone's forces are not rows of the contact frame)."""
        s = self._sim
        if int(getattr(s.model, "opt_cone", 1)) != 1:
            raise NotImplementedError("contact_force() supports elliptic friction cones (cone=\"elliptic\") only; this model uses "
                                      "pyramidal cones")
        self._require("step2")
        self._require("contacts")
        import torch

        adr, dim, ncon, f, nefc = s.contact_efc_address, s.contact_dim, s.ncon, s.efc_force, s.nefc
        mc = adr.shape[1]
        if contact is not None:
            c = int(contact)
            if not 0 <= c < mc:
                raise ValueError("contact index {} out of range [0, {})".format(c, mc))
            adr, dim = adr[:, c:c + 1], dim[:, c:c + 1]
            slot = torch.full((1,), c, device=adr.device)
        else:
            slot = torch.arange(mc, device=adr.device)
        k = torch.arange(6, device=adr.device)
        live = (adr >= 0) & (slot[None, :] < ncon[:, None].to(slot.dtype))                  # [N, C]
        # only rows below nefc: if the contact records and the rows come from different steps (one export switched on after the
        # other's last write), a stale dim must not index past the rows the solve wrote - or past efc_force itself
        row = adr[..., None].long() + k
        take = live[..., None] & (k < dim[..., None]) & (row < nefc[:, None, None].long())  # [N, C, 6]
        idx = torch.where(take, row, torch.zeros((), dtype=torch.long, device=adr.device)).clamp_(0, f.shape[1] - 1)
        out = torch.gather(f, 1, idx.reshape(idx.shape[0], -1)).reshape(idx.shape)
        out = torch.where(take, out, torch.zeros((), dtype=f.dtype, device=f.device))
        return out[:, 0] if contact is not None else out

    def full_m(self):
        """mj_fullM: the dense mass matrices [N, nv, nv] (a copy)"""
        self._require("step1")
        return self._sim.full_m()

    # ---- poses
    def _pos(self, kind, obj):
        return self._array({"body": "xpos"}.get(kind, kind + "_xpos"), "step1")[:, self._id(kind, obj)]

    def _mat(self, kind, obj):
        return self._array({"body": "xmat"}.get(kind, kind + "_xmat"), "step1")[:, self._id(kind, obj)].reshape(-1, 3, 3)

    def get_body_xpos(self, body):
        return self._pos("body", body)

    def get_body_xquat(self, body):
        return self._array("xquat", "step1")[:, self._id("body", body)]

    def get_body_xmat(self, body):
        return self._mat("body", body)

    def get_site_xpos(self, site):
        return self._pos("site", site)

    def get_site_xmat(self, site):
        return self._mat("site", site)

    def get_geom_xpos(self, geom):
        return self._pos("geom", geom)

    def get_geom_xmat(self, geom):
        return self._mat("geom", geom)

    # ---- Jacobians and point velocities
    def _jac(self, kind, obj):
        self._require("step1")
        return getattr(self._sim, "jac_" + kind)(self._id(kind, obj))

    def _vel(self, jac):
        """jac [N, 3, nv] @ qvel [N, nv] -> [N, 3]"""
        return (jac @ self._sim.qvel[:, :, None])[:, :, 0]

    def get_body_jacp(self, body):
        return self._jac("body", body)[0]

    def get_body_jacr(self, body):
        return self._jac("body", body)[1]

    def get_site_jacp(self, site):
        return self._jac("site", site)[0]

    def get_site_jacr(self, site):
        return self._jac("site", site)[1]

    def get_geom_jacp(self, geom):
        return self._jac("geom", geom)[0]

    def get_geom_jacr(self, geom):
        return self._jac("geom", geom)[1]

    def get_body_xvelp(self, body):
        return self._vel(self.get_body_jacp(body))

    def get_body_xvelr(self, body):
        return self._vel(self.get_body_jacr(body))

    def get_site_xvelp(self, site):
        return self._vel(self.get_site_jacp(site))

    def get_site_xvelr(self, site):
        return self._vel(self.get_site_jacr(site))

    def get_geom_xvelp(self, geom):
        return self._vel(self.get_geom_jacp(geom))

    def get_geom_xvelr(self, geom):
        return self._vel(self.get_geom_jacr(geom))
