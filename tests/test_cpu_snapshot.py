"""Snapshot files (state_io.save_snapshot / load_snapshot) on synthetic rows: no device needed."""
import numpy as np
import pytest

from robosuite_b200.engine import B2S_F32, B2S_F64, B2S_I32, Snapshot
from robosuite_b200.state_io import load_snapshot, save_snapshot


def _synthetic(k=3):
    sections = [("qpos", 0, 9, B2S_F32), ("warn", 48, 1, B2S_I32), ("time", 64, 1, B2S_F64), ("geom_size:12", 80, 3, B2S_F32)]
    rows = np.zeros((k, 96), dtype=np.uint8)
    rng = np.random.default_rng(0)
    for r in range(k):
        rows[r, 0:36] = rng.standard_normal(9).astype(np.float32).view(np.uint8)
        rows[r, 48:52] = np.array([r * 4], dtype=np.int32).view(np.uint8)
        rows[r, 64:72] = np.array([0.05 * r], dtype=np.float64).view(np.uint8)
        rows[r, 80:92] = np.array([0.02, 0.021, 0.022], dtype=np.float32).view(np.uint8)
    return Snapshot(rows, 0xFEDCBA9876543210, "f32", sections)


def test_round_trip(tmp_path):
    snap = _synthetic()
    extra = {"timestep": np.array([3, 4, 5]), "done": np.array([False, True, False]),
             "objects_in_bins": np.zeros((3, 4), dtype=bool)}
    p = str(tmp_path / "s.npz")
    save_snapshot(p, snap, extra=extra)
    back, ex = load_snapshot(p)
    assert back.signature == snap.signature and back.precision == "f32" and back.sections == snap.sections
    assert back.rows.dtype == np.uint8 and np.array_equal(back.rows, snap.rows)
    for name in snap.names:
        a, b = back.field(name), snap.field(name)
        assert a.dtype == b.dtype and np.array_equal(a, b), name
    assert back.field("time").dtype == np.float64 and back.field("warn")[:, 0].tolist() == [0, 4, 8]
    assert set(ex) == set(extra)
    for k, v in extra.items():
        assert ex[k].dtype == v.dtype and np.array_equal(ex[k], v), k


def test_truncated_or_mismatched_file_rejected(tmp_path):
    snap = _synthetic()
    p = str(tmp_path / "s.npz")
    save_snapshot(p, snap)
    data = open(p, "rb").read()
    cut = str(tmp_path / "cut.npz")
    with open(cut, "wb") as f:
        f.write(data[: len(data) // 2])
    with pytest.raises(ValueError):
        load_snapshot(cut)
    # rows narrower than the section table says
    narrow = Snapshot(snap.rows[:, :80].copy(), snap.signature, "f32", snap.sections)
    q = str(tmp_path / "narrow.npz")
    save_snapshot(q, narrow)
    with pytest.raises(ValueError):
        load_snapshot(q)
    # overlapping sections
    bad = Snapshot(snap.rows, snap.signature, "f32", [("qpos", 0, 9, B2S_F32), ("warn", 32, 1, B2S_I32)])
    r = str(tmp_path / "overlap.npz")
    save_snapshot(r, bad)
    with pytest.raises(ValueError):
        load_snapshot(r)
    # an npz that is not a snapshot
    other = str(tmp_path / "other.npz")
    np.savez(other, states=np.zeros((2, 3)))
    with pytest.raises(ValueError):
        load_snapshot(other)


def test_signature_mismatch_names_sections():
    from robosuite_b200.engine import snapshot_mismatch

    a = _synthetic().sections
    b = a[:3] + [("geom_size:13", 80, 3, B2S_F32), ("obs", 96, 40, B2S_F32)]
    assert snapshot_mismatch(a, b) == ["geom_size:12", "geom_size:13", "obs"]
    assert snapshot_mismatch(a, a) == []
