"""ctypes binding of libb2s.so (the C ABI in include/b2s.h) with device arrays exposed as torch.cuda tensors.

Host-side mirror of the reference's engine shim `robosuite/utils/binding_utils.py` (MjSim: from_xml_string, reset,
forward, step, step1, step2, get_state/set_state), batched over `n_env` environments.  There is no CPU fallback:
construction fails loudly when the CUDA library or a GPU is missing.
"""
import ctypes as C
import os

import numpy as np

from .errors import SimulationError
from .mjcf.compiler import Model, compile_mjcf, pack_model

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

B2S_F32, B2S_F64, B2S_I32, B2S_I64 = 0, 1, 2, 3


class B2SError(SimulationError, RuntimeError):
    """non-zero return code of the C library (message from b2s_last_error)"""


class CtrlCfg(C.Structure):
    _fields_ = [
        ("kind", C.c_int), ("action_dim", C.c_int), ("n_arm", C.c_int), ("arm_dof", C.c_int * 8),
        ("arm_qpos", C.c_int * 8), ("arm_act", C.c_int * 8), ("eef_site", C.c_int), ("base_site", C.c_int),
        ("n_grip", C.c_int), ("grip_act", C.c_int * 4), ("grip_sign", C.c_double * 4), ("grip_speed", C.c_double),
        ("kp", C.c_double * 6), ("damping_ratio", C.c_double * 6), ("input_max", C.c_double * 6),
        ("input_min", C.c_double * 6), ("output_max", C.c_double * 6), ("output_min", C.c_double * 6),
        ("null_kp", C.c_double), ("uncouple_pos_ori", C.c_int), ("n_obs_site", C.c_int),
        ("jv_kp", C.c_double * 8), ("jv_ki", C.c_double * 8), ("jv_kd", C.c_double * 8), ("jv_in_max", C.c_double * 8),
        ("jv_in_min", C.c_double * 8), ("jv_out_max", C.c_double * 8), ("jv_out_min", C.c_double * 8),
        ("jv_vel_lo", C.c_double), ("jv_vel_hi", C.c_double), ("jv_use_vel_limits", C.c_int), ("jv_torque_comp", C.c_int),
        # b2s_ctrl_cfg ends here.  Then b2s_impedance_cfg (include/b2s.h), which ctrl_config passes to b2s_ctrl_impedance:
        # IMPEDANCE_* and the clip limits of the gains taken from the action
        ("impedance_mode", C.c_int), ("kp_min", C.c_double * 8), ("kp_max", C.c_double * 8),
        ("damping_ratio_min", C.c_double * 8), ("damping_ratio_max", C.c_double * 8),
    ]


IMPEDANCE_FIXED, IMPEDANCE_VARIABLE, IMPEDANCE_VARIABLE_KP = 0, 1, 2


# per-environment model fields that are whole dof vectors (model_override(field) with no object id)
DOF_FIELDS = ("dof_damping", "dof_armature", "dof_frictionloss")
# per-environment contact parameters of a declared geom (arrays "<field>:<id>" that come with the geom's slot)
GEOM_CONTACT_FIELDS = ("geom_solref", "geom_solimp")
PERTURB_SCALE, PERTURB_SHIFT = 0, 1


CORRUPT_NONE, CORRUPT_GAUSSIAN, CORRUPT_UNIFORM = 0, 1, 2

PLACE_MAXROT = 8


class PlaceSpec(C.Structure):
    """b2s_place: one object of b2s_place_config's program (include/b2s.h)"""
    _fields_ = [("qpos_adr", C.c_int), ("body", C.c_int), ("ref", C.c_int), ("ensure_valid", C.c_int), ("axis", C.c_int),
                ("n_rot", C.c_int), ("x_min", C.c_double), ("x_max", C.c_double), ("y_min", C.c_double), ("y_max", C.c_double),
                ("base", C.c_double * 3), ("ref_dz", C.c_double), ("z_offset", C.c_double), ("bottom_dz", C.c_double),
                ("radius", C.c_double), ("bottom", C.c_double), ("top", C.c_double), ("rot_min", C.c_double * PLACE_MAXROT),
                ("rot_max", C.c_double * PLACE_MAXROT)]


class ObsMod(C.Structure):
    """b2s_obs_mod: period (s) and corruptor of one observable (b2s_obs_modifiers)"""
    _fields_ = [("period", C.c_double), ("corruptor", C.c_int), ("p0", C.c_double), ("p1", C.c_double), ("low", C.c_double),
                ("high", C.c_double)]


class PerturbSpec(C.Structure):
    """b2s_perturb: one (field, id) entry of b2s_perturb_config"""
    _fields_ = [("field", C.c_char_p), ("id", C.c_int), ("mode", C.c_int), ("amplitude", C.c_double), ("one_draw", C.c_int)]


def normalize_perturb_spec(spec):
    """perturb_config entries as (field, id, mode, amplitude, one_draw) tuples: dicts or tuples in, id None -> -1, mode names -> codes"""
    out = []
    for e in spec:
        if isinstance(e, dict):
            e = (e["field"], e.get("id"), e.get("mode", PERTURB_SCALE), e["amplitude"], e.get("one_draw", False))
        f, i, mode, amp = e[:4]
        one = e[4] if len(e) > 4 else False
        mode = {"scale": PERTURB_SCALE, "shift": PERTURB_SHIFT}.get(mode, mode)
        out.append((str(f), -1 if i is None else int(i), int(mode), float(amp), int(bool(one))))
    return out


def lib():
    global _LIB
    if _LIB is None:
        so = os.environ.get("B2S_LIB", os.path.join(_HERE, "libb2s.so"))
        if not os.path.exists(so):
            raise B2SError(f"{so} is missing: run `python -m robosuite_b200.build` (no CPU fallback exists)")
        L = C.CDLL(so)
        L.b2s_last_error.restype = C.c_char_p
        L.b2s_create.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_void_p)]
        L.b2s_destroy.argtypes = [C.c_void_p]
        L.b2s_destroy.restype = None
        L.b2s_set_stream.argtypes = [C.c_void_p, C.c_void_p]
        L.b2s_reset.argtypes = [C.c_void_p, C.c_void_p]
        for fn in ("b2s_forward", "b2s_step1", "b2s_step2"):
            getattr(L, fn).argtypes = [C.c_void_p]
        L.b2s_step.argtypes = [C.c_void_p, C.c_int]
        L.b2s_array.argtypes = [C.c_void_p, C.c_char_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int), C.POINTER(C.c_int),
                                C.POINTER(C.c_int64)]
        L.b2s_jac_site.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        L.b2s_get_state.argtypes = [C.c_void_p, C.c_void_p]
        L.b2s_set_state.argtypes = [C.c_void_p, C.c_void_p]
        L.b2s_name2id.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p]
        L.b2s_id2name.argtypes = [C.c_void_p, C.c_char_p, C.c_int]
        L.b2s_id2name.restype = C.c_char_p
        L.b2s_full_m.argtypes = [C.c_void_p, C.c_void_p]
        L.b2s_jac_body.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        L.b2s_jac_geom.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        L.b2s_ctrl_config.argtypes = [C.c_void_p, C.POINTER(CtrlCfg)]
        L.b2s_ctrl_reset.argtypes = [C.c_void_p, C.c_void_p]
        L.b2s_env_step.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        L.b2s_reset_envs.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.b2s_body_pose_override.argtypes = [C.c_void_p, C.c_int]
        L.b2s_body_pose_override_tree.argtypes = [C.c_void_p, C.c_int]
        L.b2s_model_override.argtypes = [C.c_void_p, C.c_char_p, C.c_int]
        L.b2s_set_const.argtypes = [C.c_void_p, C.c_void_p]
        L.b2s_perturb_config.argtypes = [C.c_void_p, C.POINTER(PerturbSpec), C.c_int]
        L.b2s_perturb_model.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64]
        L.b2s_place_config.argtypes = [C.c_void_p, C.POINTER(PlaceSpec), C.c_int]
        L.b2s_place_objects.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64]
        L.b2s_obs_config.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        L.b2s_obs_modifiers.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.POINTER(ObsMod), C.c_uint64]
        L.b2s_obs_objects.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        L.b2s_task_config.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int]
        L.b2s_task_config2.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int]
        L.b2s_task_objects.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        L.b2s_task_table.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        L.b2s_set_export.argtypes = [C.c_void_p, C.c_int]
        L.b2s_set_contact_export.argtypes = [C.c_void_p, C.c_int]
        L.b2s_set_step1_export.argtypes = [C.c_void_p, C.c_int]
        L.b2s_set_step2_export.argtypes = [C.c_void_p, C.c_int]
        L.b2s_set_mode.argtypes = [C.c_void_p, C.c_int]
        L.b2s_launch_count.argtypes = [C.c_void_p]
        L.b2s_launch_count.restype = C.c_int64
        L.b2s_snapshot_info.argtypes = [C.c_void_p, C.POINTER(C.c_size_t), C.POINTER(C.c_uint64), C.POINTER(C.c_int)]
        L.b2s_snapshot_section.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_int64), C.POINTER(C.c_int64),
                                           C.POINTER(C.c_int)]
        L.b2s_snapshot.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        L.b2s_restore.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        _LIB = L
    return _LIB


class _DevArray:
    """Minimal __cuda_array_interface__ carrier so torch can alias library-owned device memory without a copy."""

    def __init__(self, ptr, shape, typestr, owner):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (int(ptr), False),
                                         "version": 2, "strides": None}
        self._owner = owner


_TYPESTR = {B2S_F32: "<f4", B2S_F64: "<f8", B2S_I32: "<i4", B2S_I64: "<i8"}


_ITEMSIZE = {B2S_F32: 4, B2S_F64: 8, B2S_I32: 4, B2S_I64: 8}
_PRECISION_NAME = {B2S_F32: "f32", B2S_F64: "f64"}


class Snapshot:
    """Whole-environment snapshot rows (b2s_snapshot): `rows` uint8 [k, row_bytes] (a device tensor, or a numpy array when loaded
    from a file), `signature` (64-bit, see include/b2s.h), `precision` ("f32" / "f64") and `sections`, a list of
    (name, offset_bytes, count, dtype code) in row order.  A row holds everything that decides an environment's next control step."""

    def __init__(self, rows, signature, precision, sections):
        self.rows, self.signature, self.precision = rows, int(signature), str(precision)
        self.sections = [(str(n), int(o), int(c), int(d)) for n, o, c, d in sections]

    def __len__(self):
        return int(self.rows.shape[0])

    @property
    def names(self):
        return [s[0] for s in self.sections]

    def field(self, name):
        """typed view [k, count] of one section of every row (a torch view of the device rows, or a numpy view)"""
        for n, off, cnt, dt in self.sections:
            if n == name:
                raw = self.rows[:, off:off + cnt * _ITEMSIZE[dt]]
                if isinstance(raw, np.ndarray):
                    return raw.view(np.dtype(_TYPESTR[dt]))
                import torch

                return raw.view({B2S_F32: torch.float32, B2S_F64: torch.float64, B2S_I32: torch.int32, B2S_I64: torch.int64}[dt])
        raise KeyError("snapshot has no section %r" % name)


def snapshot_mismatch(a_sections, b_sections):
    """names of the sections that differ (present in one table only, or with another count / dtype) between two section tables"""
    a = {n: (c, d) for n, _, c, d in a_sections}
    b = {n: (c, d) for n, _, c, d in b_sections}
    return sorted(n for n in set(a) | set(b) if a.get(n) != b.get(n))


_LIVE = None  # weak set of open BatchedSim objects (a device holds at most B2S_NSLOT = 8 live handles: descriptor slots)


def close_all():
    """Destroy every live handle of this process (test teardown, interpreter exit)."""
    for sim in list(_LIVE or ()):
        sim.close()


class BatchedSim:
    """n_env independent copies of one compiled model, stepped by the per-warp CUDA engine."""

    def __init__(self, model, n_env, device=0, precision="f32", maxcon=None, maxefc=None, tier_small=None):
        import copy

        import torch

        if isinstance(model, str):
            model = compile_mjcf(model)
        assert isinstance(model, Model)
        if maxcon is not None or maxefc is not None or tier_small is not None:
            model = copy.copy(model)  # capacities travel inside the model blob: never write them into the caller's (shared) Model
            if maxcon is not None:
                model.opt_maxcon = int(maxcon)
            if maxefc is not None:
                model.opt_maxefc = int(maxefc)
            if tier_small is not None:
                # small tier of the tail kernel: capacities (contacts, constraint rows) almost every environment stays within; the
                # rest is re-run with (maxcon, maxefc) - results are the same, shared memory per warp is 2-3x smaller
                model.opt_maxcon_small, model.opt_maxefc_small = int(tier_small[0]), int(tier_small[1])
        self.model = model
        self.n_env = int(n_env)
        self.device = int(device)
        self.torch_device = torch.device("cuda", self.device)
        self.precision = B2S_F32 if precision in ("f32", "float32") else B2S_F64
        self.dtype = torch.float32 if self.precision == B2S_F32 else torch.float64
        blob = pack_model(model)
        self._h = C.c_void_p()
        self._L = lib()
        self._check(self._L.b2s_create(blob, len(blob), self.n_env, self.device, self.precision, C.byref(self._h)))
        self._cache = {}
        self.full_export = True     # set_export (the library's default)
        self.step1_export = False  # set_step1_export
        self.step2_export = False  # set_step2_export
        self.contact_export = False  # set_contact_export
        global _LIVE
        if _LIVE is None:
            import weakref

            _LIVE = weakref.WeakSet()
        _LIVE.add(self)

    def _check(self, rc):
        if rc != 0:
            raise B2SError(self._L.b2s_last_error().decode())

    def close(self):
        if getattr(self, "_h", None):
            self._L.b2s_destroy(self._h)
            self._h = None

    free = close

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def array(self, name):
        """torch tensor aliasing the named device array (leading dim n_env)."""
        import torch

        if name not in self._cache:
            ptr, dt, nd = C.c_void_p(), C.c_int(), C.c_int()
            shape = (C.c_int64 * 4)()
            self._check(self._L.b2s_array(self._h, name.encode(), C.byref(ptr), C.byref(dt), C.byref(nd), shape))
            shp = [int(shape[i]) for i in range(nd.value)]
            if any(s == 0 for s in shp):
                t = torch.zeros(shp, device=self.torch_device)
            else:
                t = torch.as_tensor(_DevArray(ptr.value, shp, _TYPESTR[dt.value], self), device=self.torch_device)
            self._cache[name] = t
        return self._cache[name]

    def __getattr__(self, name):
        if name.startswith("_"):
            raise AttributeError(name)
        try:
            return self.array(name)
        except B2SError:
            raise AttributeError(name)

    def set_stream(self, stream):
        self._check(self._L.b2s_set_stream(self._h, C.c_void_p(stream.cuda_stream if hasattr(stream, "cuda_stream") else int(stream))))

    def reset(self, mask=None):
        self._check(self._L.b2s_reset(self._h, None if mask is None else C.c_void_p(mask.data_ptr())))

    def forward(self):
        self._check(self._L.b2s_forward(self._h))

    def step1(self):
        self._check(self._L.b2s_step1(self._h))

    def step2(self):
        self._check(self._L.b2s_step2(self._h))

    def step(self, n_substeps=1):
        self._check(self._L.b2s_step(self._h, int(n_substeps)))

    def jac_site(self, site_id):
        import torch

        jp = torch.empty((self.n_env, 3, self.model.nv), dtype=self.dtype, device=self.torch_device)
        jr = torch.empty_like(jp)
        self._check(self._L.b2s_jac_site(self._h, int(site_id), C.c_void_p(jp.data_ptr()), C.c_void_p(jr.data_ptr())))
        return jp, jr

    def ctrl_config(self, cfg: CtrlCfg):
        """b2s_ctrl_config, then b2s_ctrl_impedance with the impedance block that trails the struct"""
        self._check(self._L.b2s_ctrl_config(self._h, C.byref(cfg)))
        if cfg.impedance_mode:
            self._check(self._L.b2s_ctrl_impedance(self._h, C.byref(cfg, CtrlCfg.impedance_mode.offset)))

    def reset_envs(self, mask=None, qpos=None):
        """masked episode reset entirely on the device (b2s_reset_envs): mask uint8 [n_env] or None, qpos [n_env, nq] or None (qpos0)"""
        if qpos is not None:
            assert qpos.is_cuda and qpos.dtype == self.dtype and qpos.is_contiguous() and qpos.shape == (self.n_env, self.model.nq)
        self._check(self._L.b2s_reset_envs(self._h, None if mask is None else C.c_void_p(mask.data_ptr()),
                                           None if qpos is None else C.c_void_p(qpos.data_ptr())))

    def body_pose_override(self, body_id):
        """(pos [n_env, 3], quat [n_env, 4]) tensors that replace the constant world pose of a world-welded body per environment
        (b2s_body_pose_override; the reference writes model.body_pos / body_quat per reset, door.py:417-427)"""
        self._check(self._L.b2s_body_pose_override(self._h, int(body_id)))
        return self.array("body_xpos_ov:%d" % body_id), self.array("body_xquat_ov:%d" % body_id)

    def body_pose_override_tree(self, body_id):
        """body_pose_override, and every world-welded body below it without an override of its own follows it with its fixed
        relative pose (b2s_body_pose_override_tree): a robot's welded root moved per environment"""
        self._check(self._L.b2s_body_pose_override_tree(self._h, int(body_id)))
        return self.array("body_xpos_ov:%d" % body_id), self.array("body_xquat_ov:%d" % body_id)

    def model_override(self, field, obj_id=None):
        """[n_env, ...] tensor of per-environment values of one model field for one object (b2s_model_override): "geom_size" /
        "geom_friction" [n_env, 3], "geom_solref" [n_env, 2] and "geom_solimp" [n_env, 5] of a colliding primitive geom, "body_mass"
        [n_env] / "body_inertia" [n_env, 3] (principal moments in the model's inertial frame) of a moving body, and the whole dof
        vectors "dof_damping" / "dof_armature" / "dof_frictionloss" [n_env, nv] (obj_id None).  Starts at the model's values.  The
        constants derived from these values (dof_invweight0, body_invweight0, meaninertia, the geom's bounding radius and box) follow
        at the next set_const() or reset.  A geom's solref / solimp come with its slot in the library: asking for them declares the
        geom through its friction (an array that starts at, and keeps, the model's values until written)."""
        oid = -1 if obj_id is None else int(obj_id)
        declared = "geom_friction" if field in GEOM_CONTACT_FIELDS else field
        self._check(self._L.b2s_model_override(self._h, declared.encode(), oid))
        return self.array(field if field in DOF_FIELDS else "%s:%d" % (field, oid))

    def perturb_config(self, spec):
        """configure perturb_model (b2s_perturb_config): a list of entries (field, id, mode, amplitude, one_draw) or dicts with those
        keys (id None = -1, mode "scale" / "shift" or PERTURB_SCALE / PERTURB_SHIFT, one_draw default False); every field must be
        declared with model_override first.  An empty list clears the configuration."""
        entries = normalize_perturb_spec(spec)
        arr = (PerturbSpec * max(len(entries), 1))()
        names = [f.encode() for f, *_ in entries]  # kept alive for the call
        for k, (f, i, mode, amp, one) in enumerate(entries):
            arr[k] = PerturbSpec(names[k], i, mode, amp, one)
        self._check(self._L.b2s_perturb_config(self._h, arr, len(entries)))

    def perturb_model(self, mask=None, seed=0, counter=0):
        """redraw every configured override of the masked environments (uint8 [n_env] device mask, None = all) around the model's
        values in one launch (b2s_perturb_model): Philox4x32-10 keyed by `seed`, counter (env, counter, entry, component).  The
        derived constants follow at the next set_const() or reset."""
        self._check(self._L.b2s_perturb_model(self._h, None if mask is None else C.c_void_p(mask.data_ptr()), int(seed) & (2 ** 64 - 1),
                                              int(counter)))

    def place_config(self, entries):
        """the placement program (b2s_place_config): a list of dicts with the fields of b2s_place (include/b2s.h), "rot" a list of
        (min, max) pairs; an empty list clears it"""
        arr = (PlaceSpec * max(len(entries), 1))()
        for k, e in enumerate(entries):
            rot = list(e["rot"])
            if not 1 <= len(rot) <= PLACE_MAXROT:
                raise ValueError("a placement entry takes 1 to %d rotation ranges, got %d" % (PLACE_MAXROT, len(rot)))
            pad = [0.0] * (PLACE_MAXROT - len(rot))
            arr[k] = PlaceSpec(int(e["qpos_adr"]), int(e["body"]), int(e["ref"]), int(bool(e["ensure_valid"])), int(e["axis"]), len(rot),
                               *(float(e[f]) for f in ("x_min", "x_max", "y_min", "y_max")), (C.c_double * 3)(*map(float, e["base"])),
                               *(float(e[f]) for f in ("ref_dz", "z_offset", "bottom_dz", "radius", "bottom", "top")),
                               (C.c_double * PLACE_MAXROT)(*[float(a) for a, _ in rot], *pad),
                               (C.c_double * PLACE_MAXROT)(*[float(b) for _, b in rot], *pad))
        self._check(self._L.b2s_place_config(self._h, arr, len(entries)))

    def place_objects(self, qpos, mask=None, seed=0, counter=0):
        """place the configured objects of the masked environments (uint8 [n_env] device mask, None = all) in one launch
        (b2s_place_objects): free joints into qpos (float64 [n_env, nq] on the device), world-welded bodies into their pose overrides.
        Philox4x32-10 keyed by `seed`, counter (env, counter, entry, try); an environment without a valid try for some object gets
        warn bit 1024 at the next reset_envs"""
        if qpos is not None:
            import torch

            assert qpos.is_cuda and qpos.dtype == torch.float64 and qpos.is_contiguous() and qpos.shape == (self.n_env, self.model.nq)
        self._check(self._L.b2s_place_objects(self._h, None if qpos is None else C.c_void_p(qpos.data_ptr()),
                                              None if mask is None else C.c_void_p(mask.data_ptr()), int(seed) & (2 ** 64 - 1), int(counter)))

    def set_const(self, mask=None):
        """recompute the derived constants of the masked environments (uint8 [n_env] device mask, None = all) from their
        per-environment model values, on the device (b2s_set_const); warn bit 128 marks invalid values"""
        self._check(self._L.b2s_set_const(self._h, None if mask is None else C.c_void_p(mask.data_ptr())))

    def ctrl_reset(self, mask=None):
        self._check(self._L.b2s_ctrl_reset(self._h, None if mask is None else C.c_void_p(mask.data_ptr())))

    def env_step(self, action, n_substeps):
        assert action.is_cuda and action.dtype == self.dtype and action.is_contiguous()
        self._check(self._L.b2s_env_step(self._h, C.c_void_p(action.data_ptr()), int(n_substeps)))

    def obs_config(self, ops, a, b):
        ops, a, b = (np.ascontiguousarray(x, dtype=np.int32) for x in (ops, a, b))
        self._check(self._L.b2s_obs_config(self._h, len(ops), ops.ctypes.data, a.ctypes.data, b.ctypes.data))

    def obs_modifiers(self, row_obs, mods, seed=0):
        """sampling rates and corruptors of the observables (b2s_obs_modifiers): row_obs [obs_dim] = the observable of each observation
        row, mods = one (period_s, corruptor, p0, p1, low, high) per observable (corruptor CORRUPT_NONE / GAUSSIAN (p0 mean, p1 std) /
        UNIFORM (p0 min_noise, p1 max_noise)), noise keyed by `seed`.  Empty `mods` clears the configuration.  The per-environment
        timers, flags and sample counts are the arrays "obs_timer", "obs_sampled" and "obs_nsample"."""
        mods = list(mods)
        rows = np.ascontiguousarray(row_obs, dtype=np.int32)
        arr = (ObsMod * max(len(mods), 1))()
        for k, (T, kind, p0, p1, lo, hi) in enumerate(mods):
            arr[k] = ObsMod(float(T), int(kind), float(p0), float(p1), float(lo), float(hi))
        self._check(self._L.b2s_obs_modifiers(self._h, len(mods), rows.ctypes.data if len(mods) else None, arr,
                                              int(seed) & (2 ** 64 - 1)))
        for name in ("obs_timer", "obs_sampled", "obs_nsample"):  # arrays may have been (re)created
            self._cache.pop(name, None)

    def obs_objects(self, body_ids):
        """per-environment object selection (b2s_obs_objects): 1 to 4 bodies with a free joint.  Returns the "obj_sel" tensor [n_env]
        int32 (zeros when first created): the observation / task ops OB_SEL_* of environment e read body body_ids[obj_sel[e]].  An
        empty list clears the selection (B2SError while a table still reads it) and returns None."""
        ids = np.ascontiguousarray(body_ids, dtype=np.int32).reshape(-1)
        self._check(self._L.b2s_obs_objects(self._h, len(ids), ids.ctypes.data if len(ids) else None))
        return self.array("obj_sel") if len(ids) else None

    def task_config(self, body, site, left, right, obj):
        left, right, obj = (np.ascontiguousarray(x, dtype=np.int32) for x in (left, right, obj))
        self._check(self._L.b2s_task_config(self._h, int(body), int(site), left.ctypes.data, len(left), right.ctypes.data,
                                            len(right), obj.ctypes.data, len(obj)))

    def task_config2(self, body2, obj2):
        obj2 = np.ascontiguousarray(obj2, dtype=np.int32)
        self._check(self._L.b2s_task_config2(self._h, int(body2), obj2.ctypes.data, len(obj2)))

    def task_table(self, rows):
        """rows: [(op, a, b), ...] in the observation-table encoding -> array `task_vec` [n_env, len(rows)]"""
        arr = np.ascontiguousarray(rows, dtype=np.int32).reshape(-1, 3)
        op, a, b = (np.ascontiguousarray(arr[:, k]) for k in range(3))
        self._check(self._L.b2s_task_table(self._h, len(op), op.ctypes.data, a.ctypes.data, b.ctypes.data))

    def task_objects(self, geom_lists):
        """per-object grasp flags (task_out[:, 5] = bit i set when object i is grasped); at most 4 objects"""
        flat = np.ascontiguousarray([g for l in geom_lists for g in l], dtype=np.int32)
        cnt = np.ascontiguousarray([len(l) for l in geom_lists], dtype=np.int32)
        self._check(self._L.b2s_task_objects(self._h, len(geom_lists), flat.ctypes.data, cnt.ctypes.data))

    def set_export(self, flag):
        """whether b2s_env_step also writes the derived arrays (xpos, contacts, ...) of its last substep to HBM"""
        self._check(self._L.b2s_set_export(self._h, int(bool(flag))))
        self.full_export = bool(flag)

    # the array-group exports: the library's setter and the attribute that records the flag
    _EXPORTS = {"contacts": ("b2s_set_contact_export", "contact_export"), "step1": ("b2s_set_step1_export", "step1_export"),
                "step2": ("b2s_set_step2_export", "step2_export")}

    def _set_group_export(self, group, flag):
        fn, attr = self._EXPORTS[group]
        self._check(getattr(self._L, fn)(self._h, int(bool(flag))))
        setattr(self, attr, bool(flag))

    def set_step1_export(self, flag):
        """whether the last substep of every env_step / step writes the step-1 arrays (xpos, xquat, xmat, site / colliding-geom
        poses, qM, cdof, qfrc_bias, qfrc_passive: what `data` reads) in every mode, without the rest of the derived-array export
        (b2s_set_step1_export)"""
        self._set_group_export("step1", flag)

    def set_step2_export(self, flag):
        """whether the last substep of every env_step / step writes the step-2 arrays (qfrc_actuator, actuator_force, qfrc_smooth,
        qacc_smooth, qfrc_constraint, nefc, efc_*, solver_niter, contact_efc_address: what `data`'s dynamics properties and
        contact_force() read) in every mode, without the rest of the derived-array export (b2s_set_step2_export)"""
        self._set_group_export("step2", flag)

    @property
    def data(self):
        """the batched MjData view of the step-1 and step-2 arrays (robosuite_b200/data.py); after env_step / step it needs
        set_step1_export(True) (poses, Jacobians, mass matrices), set_step2_export(True) (forces, constraint rows; contact_force()
        also set_contact_export(True)) or set_export(True)"""
        if "_data" not in self.__dict__:
            from .data import BatchedData

            self._data = BatchedData(self)
        return self._data

    def set_contact_export(self, flag):
        """whether the last substep of every env_step / step writes the contact arrays (contacts()) in every mode, without the
        rest of the derived-array export (b2s_set_contact_export)"""
        self._set_group_export("contacts", flag)

    def contacts(self):
        """device views of the contacts of the last substep: "ncon" [N], "geom" [N, maxcon, 2] (-1 beyond ncon), "dist"
        [N, maxcon], "pos" [N, maxcon, 3], "frame" [N, maxcon, 9] (normal first) and "friction" [N, maxcon, 3].  Written by
        env_step / step with set_contact_export(True) or set_export(True), and by forward / reset_envs (masked environments)"""
        return {k: self.array(a) for k, a in (("ncon", "ncon"), ("geom", "contact_geom"), ("dist", "contact_dist"),
                                              ("pos", "contact_pos"), ("frame", "contact_frame"), ("friction", "contact_friction"))}

    def set_mode(self, mode):
        """0 = fused single kernel, 1 = pipelined phase kernels, 2 = unit queue (one persistent kernel per control step);
        identical results"""
        self._check(self._L.b2s_set_mode(self._h, int(mode)))

    @property
    def launch_count(self):
        return int(self._L.b2s_launch_count(self._h))

    # ---- whole-environment snapshots (b2s_snapshot / b2s_restore)
    def snapshot_layout(self):
        """(row_bytes, signature, sections) of this handle's snapshot rows as they are now"""
        rb, sig, ns = C.c_size_t(), C.c_uint64(), C.c_int()
        self._check(self._L.b2s_snapshot_info(self._h, C.byref(rb), C.byref(sig), C.byref(ns)))
        cached = self.__dict__.get("_snap_layout")
        if cached is not None and cached[1] == sig.value:  # the signature covers the section table: unchanged
            return cached
        secs = []
        for k in range(ns.value):
            nm, off, cnt, dt = C.c_char_p(), C.c_int64(), C.c_int64(), C.c_int()
            self._check(self._L.b2s_snapshot_section(self._h, k, C.byref(nm), C.byref(off), C.byref(cnt), C.byref(dt)))
            secs.append((nm.value.decode(), off.value, cnt.value, dt.value))
        self._snap_layout = (int(rb.value), int(sig.value), secs)
        return self._snap_layout

    def snapshot(self, env_ids=None):
        """Snapshot of environments `env_ids` (host list / array of indices, None = all in order): row r holds environment env_ids[r].
        Enqueued on the handle's stream; an index out of range raises B2SError."""
        import torch

        rb, sig, secs = self.snapshot_layout()
        if env_ids is None:
            idx, k = None, self.n_env
        else:
            idx = np.ascontiguousarray(np.asarray(env_ids.cpu() if torch.is_tensor(env_ids) else env_ids, dtype=np.int32).reshape(-1))
            k = len(idx)
        rows = torch.empty((k, rb), dtype=torch.uint8, device=self.torch_device)
        self._check(self._L.b2s_snapshot(self._h, C.c_void_p(rows.data_ptr()), None if idx is None else idx.ctypes.data, k))
        return Snapshot(rows, sig, _PRECISION_NAME[self.precision], secs)

    def restore(self, snap, src=None):
        """Environment e takes row src[e] of `snap` (-1 keeps it; src None: row e, needs len(snap) == n_env).  src: a device int32
        tensor [n_env] (used as is, e.g. an argmax computed on the device) or host indices.  A device entry >= len(snap) or < -1
        leaves its environment untouched and sets warn bit 256.  No physics runs: the exported derived arrays stay stale until the
        next forward / step.  ValueError when the snapshot's signature differs from this handle's."""
        import torch

        rb, sig, secs = self.snapshot_layout()
        if snap.signature != sig:
            diff = snapshot_mismatch(snap.sections, secs)
            why = ("sections differ: " + ", ".join(diff)) if diff else \
                "same sections, but the model, precision, controller kind or observation / task tables differ"
            raise ValueError("snapshot signature %#018x does not match this handle's %#018x (%s)" % (snap.signature, sig, why))
        rows = snap.rows
        if not torch.is_tensor(rows) or rows.device != self.torch_device:
            rows = torch.as_tensor(np.asarray(rows) if not torch.is_tensor(rows) else rows, dtype=torch.uint8).to(self.torch_device)
        rows = rows.contiguous()
        assert rows.dtype == torch.uint8 and rows.ndim == 2 and rows.shape[1] == rb
        if src is not None:
            if torch.is_tensor(src) and src.is_cuda:
                src = src.to(device=self.torch_device, dtype=torch.int32).contiguous()
            else:
                src = torch.as_tensor(np.asarray(src.cpu() if torch.is_tensor(src) else src, dtype=np.int32), device=self.torch_device)
            assert src.shape == (self.n_env,), "src must hold one source row (or -1) per environment"
        self._restore_keep = (rows, src)  # alive until the next restore: the copy runs asynchronously on the handle's stream
        self._check(self._L.b2s_restore(self._h, C.c_void_p(rows.data_ptr()), int(rows.shape[0]),
                                        None if src is None else C.c_void_p(src.data_ptr())))

    def clone_envs(self, src):
        """environment e takes the current state of environment src[e] (-1 keeps its own): snapshot of all, then restore"""
        self.restore(self.snapshot(), src)

    # ---- MjSim-style state I/O (binding_utils.py:1155-1184): flattened [time, qpos, qvel] per env
    def get_state(self):
        import torch

        out = torch.empty((self.n_env, 1 + self.model.nq + self.model.nv), dtype=self.dtype, device=self.torch_device)
        self._check(self._L.b2s_get_state(self._h, C.c_void_p(out.data_ptr())))
        return out

    def set_state(self, flat):
        flat = flat.to(device=self.torch_device, dtype=self.dtype).contiguous()
        assert flat.shape == (self.n_env, 1 + self.model.nq + self.model.nv)
        self._check(self._L.b2s_set_state(self._h, C.c_void_p(flat.data_ptr())))

    # ---- MjModel name tables / mj_fullM / body and geom Jacobians (binding_utils.py:362-492, 853-878; controller.py:226-229)
    def name2id(self, objtype, name):
        return int(self._L.b2s_name2id(self._h, objtype.encode(), name.encode()))

    def id2name(self, objtype, idx):
        r = self._L.b2s_id2name(self._h, objtype.encode(), int(idx))
        return None if r is None else r.decode()

    def full_m(self):
        import torch

        out = torch.empty((self.n_env, self.model.nv, self.model.nv), dtype=self.dtype, device=self.torch_device)
        self._check(self._L.b2s_full_m(self._h, C.c_void_p(out.data_ptr())))
        return out

    def _jac(self, fn, idx):
        import torch

        jp = torch.empty((self.n_env, 3, self.model.nv), dtype=self.dtype, device=self.torch_device)
        jr = torch.empty_like(jp)
        self._check(fn(self._h, int(idx), C.c_void_p(jp.data_ptr()), C.c_void_p(jr.data_ptr())))
        return jp, jr

    def jac_body(self, body_id):
        return self._jac(self._L.b2s_jac_body, body_id)

    def jac_geom(self, geom_id):
        return self._jac(self._L.b2s_jac_geom, geom_id)
