"""GPU: the drop-in boundary itself - libb2s's C ABI driven through ctypes WITHOUT the Python engine layer (only the blob packer and
torch for device memory), as a maintainer of the reference would bind it behind `robosuite/utils/binding_utils.py` (INTEGRATION.md).

* name tables, state I/O, mj_fullM, body / geom / site Jacobians against the compiled model and the oracle;
* two live handles of the same task stepping CONCURRENTLY on two CUDA streams (each handle owns a constant-memory descriptor slot):
  bit-identical to each other and to a handle stepped alone - round 1 kept one set of descriptors per device and could not."""
import ctypes as C
import os

import numpy as np
import pytest

from tests.schedules import switches
from tests.util import ROOT, lift_states, load

pytestmark = pytest.mark.gpu


class CtrlCfg(C.Structure):  # b2s_ctrl_cfg, include/b2s.h
    _fields_ = [
        ("kind", C.c_int), ("action_dim", C.c_int), ("n_arm", C.c_int), ("arm_dof", C.c_int * 8), ("arm_qpos", C.c_int * 8),
        ("arm_act", C.c_int * 8), ("eef_site", C.c_int), ("base_site", C.c_int), ("n_grip", C.c_int), ("grip_act", C.c_int * 4),
        ("grip_sign", C.c_double * 4), ("grip_speed", C.c_double), ("kp", C.c_double * 6), ("damping_ratio", C.c_double * 6),
        ("input_max", C.c_double * 6), ("input_min", C.c_double * 6), ("output_max", C.c_double * 6), ("output_min", C.c_double * 6),
        ("null_kp", C.c_double), ("uncouple_pos_ori", C.c_int), ("n_obs_site", C.c_int),
        ("jv_kp", C.c_double * 8), ("jv_ki", C.c_double * 8), ("jv_kd", C.c_double * 8), ("jv_in_max", C.c_double * 8),
        ("jv_in_min", C.c_double * 8), ("jv_out_max", C.c_double * 8), ("jv_out_min", C.c_double * 8),
        ("jv_vel_lo", C.c_double), ("jv_vel_hi", C.c_double), ("jv_use_vel_limits", C.c_int), ("jv_torque_comp", C.c_int)]


def _lib():
    L = C.CDLL(os.environ.get("B2S_LIB", os.path.join(ROOT, "robosuite_b200", "libb2s.so")))
    L.b2s_last_error.restype = C.c_char_p
    L.b2s_create.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_void_p)]
    L.b2s_destroy.argtypes = [C.c_void_p]; L.b2s_destroy.restype = None
    L.b2s_array.argtypes = [C.c_void_p, C.c_char_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int64)]
    for fn in ("b2s_forward",):
        getattr(L, fn).argtypes = [C.c_void_p]
    L.b2s_set_stream.argtypes = [C.c_void_p, C.c_void_p]
    L.b2s_set_mode.argtypes = [C.c_void_p, C.c_int]
    L.b2s_set_export.argtypes = [C.c_void_p, C.c_int]
    L.b2s_ctrl_config.argtypes = [C.c_void_p, C.POINTER(CtrlCfg)]
    L.b2s_ctrl_reset.argtypes = [C.c_void_p, C.c_void_p]
    L.b2s_env_step.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    L.b2s_get_state.argtypes = [C.c_void_p, C.c_void_p]
    L.b2s_set_state.argtypes = [C.c_void_p, C.c_void_p]
    L.b2s_name2id.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p]
    L.b2s_id2name.argtypes = [C.c_void_p, C.c_char_p, C.c_int]; L.b2s_id2name.restype = C.c_char_p
    L.b2s_full_m.argtypes = [C.c_void_p, C.c_void_p]
    for fn in ("b2s_jac_site", "b2s_jac_body", "b2s_jac_geom"):
        getattr(L, fn).argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    return L


class _Dev:
    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (int(ptr), False), "version": 2, "strides": None}


def _arr(L, h, name):
    import torch

    ptr, dt, nd = C.c_void_p(), C.c_int(), C.c_int()
    shape = (C.c_int64 * 4)()
    assert L.b2s_array(h, name.encode(), C.byref(ptr), C.byref(dt), C.byref(nd), shape) == 0, L.b2s_last_error()
    return torch.as_tensor(_Dev(ptr.value, [int(shape[i]) for i in range(nd.value)], {0: "<f4", 1: "<f8", 2: "<i4", 3: "<i8"}[dt.value]), device="cuda")


def _create(L, blob, n, prec=0):
    h = C.c_void_p()
    assert L.b2s_create(blob, len(blob), n, 0, prec, C.byref(h)) == 0, L.b2s_last_error()
    return h


def _lift_osc_cfg(L, h):
    """controllers/config/robots/default_panda.json + parts/osc_pose.json, indices resolved through the library's own name tables"""
    c = CtrlCfg()
    c.kind, c.action_dim, c.n_arm, c.n_grip = 1, 7, 7, 2
    q_adr = _arr(L, h, "qpos")  # only to know nq
    for k in range(7):
        j = L.b2s_name2id(h, b"joint", ("robot0_joint%d" % (k + 1)).encode())
        assert j >= 0
        c.arm_dof[k], c.arm_qpos[k] = j, j  # Lift/Panda: the arm's hinge joints are joints 0..6, one dof / one qpos each, in order
        c.arm_act[k] = L.b2s_name2id(h, b"actuator", ("robot0_torq_j%d" % (k + 1)).encode())
        assert c.arm_act[k] >= 0
    c.eef_site = L.b2s_name2id(h, b"site", b"gripper0_right_grip_site")
    c.base_site = L.b2s_name2id(h, b"site", b"robot0_right_center")
    c.grip_act[0] = L.b2s_name2id(h, b"actuator", b"gripper0_right_gripper_finger_joint1")
    c.grip_act[1] = L.b2s_name2id(h, b"actuator", b"gripper0_right_gripper_finger_joint2")
    assert min(c.eef_site, c.base_site, c.grip_act[0], c.grip_act[1]) >= 0
    c.grip_sign[0], c.grip_sign[1], c.grip_speed = -1.0, 1.0, 0.2
    for k in range(6):
        c.kp[k], c.damping_ratio[k], c.input_max[k], c.input_min[k] = 150.0, 1.0, 1.0, -1.0
        c.output_max[k], c.output_min[k] = (0.05, -0.05) if k < 3 else (0.5, -0.5)
    c.null_kp, c.uncouple_pos_ori = 10.0, 1
    return c


def test_name_tables_state_io_full_m_and_jacobians():
    import torch

    from oracle.pyoracle import Oracle
    from robosuite_b200.mjcf.compiler import pack_model

    L = _lib()
    model = load("Lift_Panda")
    blob = pack_model(model)
    n = 4
    for prec, tol in ((1, 1e-12), (0, 3e-6)):
        h = _create(L, blob, n, prec)
        dt = torch.float64 if prec else torch.float32
        # name tables agree with the compiled model in both directions
        for ty in ("body", "joint", "geom", "site", "actuator"):
            for i, nm in enumerate(model.names[ty]):
                got = L.b2s_id2name(h, ty.encode(), i)
                assert got is not None and got.decode() == ("" if nm is None else nm), (ty, i, got, nm)
                if nm:
                    assert L.b2s_name2id(h, ty.encode(), nm.encode()) == model.names[ty].index(nm)
            assert L.b2s_id2name(h, ty.encode(), len(model.names[ty])) is None
        assert L.b2s_name2id(h, b"body", b"no_such_body") == -1 and L.b2s_name2id(h, b"nonsense", b"x") == -1
        # state I/O round trip (MjSimState.flatten layout: time, qpos, qvel)
        q, v = lift_states(model, n, seed=9, vel=0.3)
        flat = torch.as_tensor(np.concatenate([np.arange(n)[:, None] * 0.5, q, v], axis=1), dtype=dt, device="cuda").contiguous()
        assert L.b2s_set_state(h, C.c_void_p(flat.data_ptr())) == 0
        back = torch.empty_like(flat)
        assert L.b2s_get_state(h, C.c_void_p(back.data_ptr())) == 0
        torch.cuda.synchronize()
        assert torch.equal(back, flat)
        assert torch.equal(_arr(L, h, "qpos"), flat[:, 1:1 + model.nq]) and torch.equal(_arr(L, h, "time"), flat[:, 0])
        # forward, then mj_fullM and Jacobians vs the oracle
        assert L.b2s_forward(h) == 0
        M = torch.empty((n, model.nv, model.nv), dtype=dt, device="cuda")
        assert L.b2s_full_m(h, C.c_void_p(M.data_ptr())) == 0
        o = Oracle(blob)
        body = model.names["body"].index("robot0_right_hand")
        geom = model.names["geom"].index("cube_g0")
        site = model.names["site"].index("gripper0_right_grip_site")
        jb = [torch.empty((n, 3, model.nv), dtype=dt, device="cuda") for _ in range(6)]
        assert L.b2s_jac_body(h, body, C.c_void_p(jb[0].data_ptr()), C.c_void_p(jb[1].data_ptr())) == 0
        assert L.b2s_jac_geom(h, geom, C.c_void_p(jb[2].data_ptr()), C.c_void_p(jb[3].data_ptr())) == 0
        assert L.b2s_jac_site(h, site, C.c_void_p(jb[4].data_ptr()), C.c_void_p(jb[5].data_ptr())) == 0
        torch.cuda.synchronize()
        for e in range(n):
            o.qpos[:] = q[e]; o.qvel[:] = v[e]; o.forward()
            assert np.abs(M[e].cpu().numpy() - o.M).max() < tol * max(1.0, np.abs(o.M).max())
            for (jp, jr), (pt, b) in zip(((jb[0], jb[1]), (jb[2], jb[3]), (jb[4], jb[5])),
                                         ((o.xpos[body], body), (o.geom_xpos[geom], int(model.geom_bodyid[geom])), (o.site_xpos[site], int(model.site_bodyid[site])))):
                ojp, ojr = o.jac(pt, b)
                assert np.abs(jp[e].cpu().numpy() - ojp).max() < tol and np.abs(jr[e].cpu().numpy() - ojr).max() < tol, (prec, e)
        L.b2s_destroy(h)


def test_two_handles_step_concurrently_and_bit_exactly():
    import torch

    from robosuite_b200.mjcf.compiler import pack_model

    L = _lib()
    model = load("Lift_Panda")
    blob = pack_model(model)
    n, steps = 64, 12
    q, _ = lift_states(model, n, seed=31)
    rng = np.random.default_rng(4)
    acts = rng.uniform(-1, 1, size=(steps, n, 7))
    acts[:, : n // 2, 2] = -1.0  # half of the arms press down: contacts, EPA, large-tier environments
    acts[:, :, 6] = 1.0
    acts_d = torch.as_tensor(acts, dtype=torch.float32, device="cuda")

    def setup(stream):
        h = _create(L, blob, n, 0)
        if stream is not None:
            assert L.b2s_set_stream(h, C.c_void_p(stream.cuda_stream)) == 0
        c = _lift_osc_cfg(L, h)
        assert L.b2s_ctrl_config(h, C.byref(c)) == 0
        assert L.b2s_set_export(h, 0) == 0 and L.b2s_set_mode(h, int(os.environ.get("B2S_TEST_MODE", "1"))) == 0
        with torch.cuda.stream(stream) if stream is not None else torch.cuda.stream(torch.cuda.current_stream()):
            _arr(L, h, "qpos").copy_(torch.as_tensor(q, dtype=torch.float32))
            assert L.b2s_forward(h) == 0 and L.b2s_ctrl_reset(h, None) == 0
        return h

    with switches(gjk_cache=False):
        sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
        ha, hb = setup(sa), setup(sb)
        torch.cuda.synchronize()
        for t in range(steps):  # interleaved enqueue: both handles' graphs are in flight at the same time
            with torch.cuda.stream(sa):
                assert L.b2s_env_step(ha, C.c_void_p(acts_d[t].data_ptr()), 25) == 0, L.b2s_last_error()
            if os.environ.get("B2S_TEST_SEQ"):
                torch.cuda.synchronize()
            with torch.cuda.stream(sb):
                assert L.b2s_env_step(hb, C.c_void_p(acts_d[t].data_ptr()), 25) == 0, L.b2s_last_error()
            if os.environ.get("B2S_TEST_SEQ"):
                torch.cuda.synchronize()
        torch.cuda.synchronize()
        qa, qb = _arr(L, ha, "qpos").clone(), _arr(L, hb, "qpos").clone()
        va, vb = _arr(L, ha, "qvel").clone(), _arr(L, hb, "qvel").clone()
        assert int(_arr(L, ha, "warn").abs().max()) == 0
        L.b2s_destroy(ha); L.b2s_destroy(hb)
        hc = setup(None)
        for t in range(steps):
            assert L.b2s_env_step(hc, C.c_void_p(acts_d[t].data_ptr()), 25) == 0
        torch.cuda.synchronize()
        qc, vc = _arr(L, hc, "qpos").clone(), _arr(L, hc, "qvel").clone()
        L.b2s_destroy(hc)
    assert torch.isfinite(qa).all()

    def where(x, y):
        return torch.nonzero((x != y).any(1)).flatten().tolist()

    assert torch.equal(qa, qb) and torch.equal(va, vb), ("two concurrent handles diverged", where(qa, qb), "A vs alone", where(qa, qc), "B vs alone", where(qb, qc))
    assert torch.equal(qa, qc) and torch.equal(va, vc), ("a handle stepped beside another differs from one stepped alone", where(qa, qc))
