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
environments had before until the next step."""


class BatchedData:
    """The batched MjData of a BatchedSim (or a stand-in with the same surface: the named arrays as attributes, jac_site /
    jac_body / jac_geom, full_m, `model`, and the `full_export` / `step1_export` flags)."""

    def __init__(self, sim):
        self._sim = sim
        m = sim.model
        self._count = {"body": int(m.nbody), "site": int(m.nsite), "geom": int(m.ngeom)}
        self._colliding = {int(g) for p in m.pair_geom for g in p}

    def _check(self):
        s = self._sim
        if not (s.full_export or s.step1_export):
            raise RuntimeError("sim.data reads the step-1 arrays, which env_step / step write only with the step-1 export on: create "
                               "the environment with make(..., data_queries=True) or call BatchedSim.set_step1_export(True)")

    def _array(self, name):
        self._check()
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
    body_xpos = property(lambda self: self._array("xpos"))
    body_xquat = property(lambda self: self._array("xquat"))
    body_xmat = property(lambda self: self._array("xmat"))
    site_xpos = property(lambda self: self._array("site_xpos"))
    site_xmat = property(lambda self: self._array("site_xmat"))
    geom_xpos = property(lambda self: self._array("geom_xpos"))
    geom_xmat = property(lambda self: self._array("geom_xmat"))
    qM = property(lambda self: self._array("qM"))
    cdof = property(lambda self: self._array("cdof"))
    qfrc_bias = property(lambda self: self._array("qfrc_bias"))
    qfrc_passive = property(lambda self: self._array("qfrc_passive"))

    def full_m(self):
        """mj_fullM: the dense mass matrices [N, nv, nv] (a copy)"""
        self._check()
        return self._sim.full_m()

    # ---- poses
    def _pos(self, kind, obj):
        return self._array({"body": "xpos"}.get(kind, kind + "_xpos"))[:, self._id(kind, obj)]

    def _mat(self, kind, obj):
        return self._array({"body": "xmat"}.get(kind, kind + "_xmat"))[:, self._id(kind, obj)].reshape(-1, 3, 3)

    def get_body_xpos(self, body):
        return self._pos("body", body)

    def get_body_xquat(self, body):
        return self._array("xquat")[:, self._id("body", body)]

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
        self._check()
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
