"""State / demonstration file formats of the reference, for batches.

* `MjSimState.flatten` layout (utils/binding_utils.py:221-249): [time, qpos(nq), qvel(nv)] per environment - what
  `BatchedSim.get_state()` / `set_state()` exchange as [N, 1 + nq + nv].
* `DataCollectionWrapper` episode folders (wrappers/data_collection_wrapper.py:100-147): `model.xml`, `ep_meta.json` and
  `state_*.npz` with `states` [T, 1 + nq + nv], `action_infos` (list of {"actions": a}), `successful`, `env`.
  `save_episodes` writes one such folder per environment of a batched rollout, `load_episode` reads one back (also folders
  written by the reference itself), so recorded demonstrations can be replayed on either side with `set_state`.
* Whole-environment snapshots (`BatchedSim.snapshot`, include/b2s.h): `save_snapshot` / `load_snapshot` keep the rows, the
  signature, the precision and the section table in one `.npz`, plus optional environment-layer arrays (`extra`).

Host-side numpy only; nothing here touches the GPU."""
import json
import os

import numpy as np


def flatten_state(time, qpos, qvel):
    """(time [N] or scalar, qpos [N, nq], qvel [N, nv]) -> [N, 1 + nq + nv]   (MjSimState.flatten per row)"""
    qpos, qvel = np.atleast_2d(np.asarray(qpos, dtype=np.float64)), np.atleast_2d(np.asarray(qvel, dtype=np.float64))
    t = np.broadcast_to(np.asarray(time, dtype=np.float64).reshape(-1, 1), (qpos.shape[0], 1))
    return np.concatenate([t, qpos, qvel], axis=1)


def unflatten_state(flat, nq, nv):
    """[N, 1 + nq + nv] (or one row) -> (time [N], qpos [N, nq], qvel [N, nv])   (MjSimState.from_flattened)"""
    flat = np.atleast_2d(np.asarray(flat, dtype=np.float64))
    if flat.shape[1] != 1 + nq + nv:
        raise ValueError("state row has %d entries, expected 1 + nq + nv = %d" % (flat.shape[1], 1 + nq + nv))
    return flat[:, 0], flat[:, 1:1 + nq], flat[:, 1 + nq:]


def save_episodes(directory, env_name, model_xml, states, actions, successful=None, ep_meta=None, prefix="ep"):
    """states [T + 1, N, 1 + nq + nv] (initial state first, as the reference records it), actions [T, N, action_dim]
    -> N folders `<directory>/<prefix>_<env index>/` in the DataCollectionWrapper layout; returns their paths"""
    states, actions = np.asarray(states), np.asarray(actions)
    if states.ndim != 3 or actions.ndim != 3 or states.shape[0] != actions.shape[0] + 1 or states.shape[1] != actions.shape[1]:
        raise ValueError("expected states [T + 1, N, D] and actions [T, N, A]")
    n = states.shape[1]
    succ = np.zeros(n, dtype=bool) if successful is None else np.asarray(successful, dtype=bool).reshape(n)
    out = []
    for e in range(n):
        ep = os.path.join(directory, "%s_%06d" % (prefix, e))
        os.makedirs(ep, exist_ok=False)
        with open(os.path.join(ep, "model.xml"), "w") as f:
            f.write(model_xml)
        with open(os.path.join(ep, "ep_meta.json"), "w") as f:
            json.dump(ep_meta or {}, f)
        np.savez(os.path.join(ep, "state_0_0.npz"), states=states[:, e], action_infos=[{"actions": a} for a in actions[:, e]],
                 successful=bool(succ[e]), env=env_name)
        out.append(ep)
    return out


def load_episode(ep_directory):
    """-> dict(model_xml, states [T', D], actions [T, A], successful, env, ep_meta); concatenates all state_*.npz files of the
    folder in name order like scripts/playback_demonstrations_from_hdf5.py's source data was gathered"""
    files = sorted(f for f in os.listdir(ep_directory) if f.startswith("state_") and f.endswith(".npz"))
    if not files:
        raise FileNotFoundError("no state_*.npz in " + ep_directory)
    states, actions, successful, env = [], [], False, None
    for f in files:
        d = np.load(os.path.join(ep_directory, f), allow_pickle=True)
        states.append(np.asarray(d["states"]))
        actions += [np.asarray(ai["actions"]) for ai in d["action_infos"]]
        successful = successful or bool(d["successful"])
        env = str(d["env"])
    xml_path, meta_path = os.path.join(ep_directory, "model.xml"), os.path.join(ep_directory, "ep_meta.json")
    xml = open(xml_path).read() if os.path.exists(xml_path) else None
    meta = json.load(open(meta_path)) if os.path.exists(meta_path) else {}
    return dict(model_xml=xml, states=np.concatenate(states, axis=0), actions=np.array(actions), successful=successful, env=env,
                ep_meta=meta)


SNAPSHOT_FORMAT = "b2s-snapshot-1"


def _check_sections(row_bytes, names, offsets, counts, dtypes):
    """section table sanity: 16-byte aligned, disjoint, inside the row"""
    from .engine import _ITEMSIZE

    if row_bytes % 16:
        raise ValueError("snapshot rows are %d bytes, not a multiple of 16" % row_bytes)
    end = 0
    for n, o, c, d in zip(names, offsets, counts, dtypes):
        if int(d) not in _ITEMSIZE or o % 16 or o < end or c < 0 or o + c * _ITEMSIZE[int(d)] > row_bytes:
            raise ValueError("snapshot section %r (offset %d, count %d, dtype %d) does not fit the row layout" % (n, o, c, d))
        end = o + c * _ITEMSIZE[int(d)]


def save_snapshot(path, snap, extra=None):
    """Write a Snapshot (rows copied to the host) and optional named arrays `extra` (e.g. the environment layer's episode clocks and
    task tensors, numpy or torch) to one .npz file."""
    rows = snap.rows.cpu().numpy() if hasattr(snap.rows, "cpu") else np.asarray(snap.rows)
    rows = np.ascontiguousarray(rows, dtype=np.uint8)
    names = [n for n, *_ in snap.sections]
    if any("\n" in n for n in names):
        raise ValueError("section names must not contain newlines")
    arrays = {"format": np.array(SNAPSHOT_FORMAT), "rows": rows, "signature": np.array(snap.signature, dtype=np.uint64),
              "precision": np.array(snap.precision), "section_names": np.array("\n".join(names)),
              "section_offsets": np.array([s[1] for s in snap.sections], dtype=np.int64),
              "section_counts": np.array([s[2] for s in snap.sections], dtype=np.int64),
              "section_dtypes": np.array([s[3] for s in snap.sections], dtype=np.int32)}
    for k, v in (extra or {}).items():
        arrays["extra/" + k] = np.asarray(v.cpu() if hasattr(v, "cpu") else v)
    with open(path, "wb") as f:
        np.savez(f, **arrays)


def load_snapshot(path):
    """-> (Snapshot with host rows, dict of the `extra` arrays).  ValueError for a file that is truncated, not a snapshot, or whose rows
    and section table disagree."""
    import zipfile

    from .engine import Snapshot

    try:
        with np.load(path, allow_pickle=False) as d:
            z = {k: d[k] for k in d.files}
    except (zipfile.BadZipFile, OSError, EOFError, ValueError) as e:
        raise ValueError("%s is not a readable snapshot file: %s" % (path, e)) from None
    need = ("format", "rows", "signature", "precision", "section_names", "section_offsets", "section_counts", "section_dtypes")
    missing = [k for k in need if k not in z]
    if missing or str(z["format"]) != SNAPSHOT_FORMAT:
        raise ValueError("%s is not a %s file (missing: %s)" % (path, SNAPSHOT_FORMAT, ", ".join(missing) or "-"))
    rows = z["rows"]
    names = str(z["section_names"]).split("\n") if str(z["section_names"]) else []
    offs, cnts, dts = (z[k].astype(np.int64).tolist() for k in ("section_offsets", "section_counts", "section_dtypes"))
    if rows.dtype != np.uint8 or rows.ndim != 2 or not (len(names) == len(offs) == len(cnts) == len(dts)):
        raise ValueError("%s: rows or section table malformed" % path)
    _check_sections(int(rows.shape[1]), names, offs, cnts, dts)
    snap = Snapshot(rows, int(z["signature"]), str(z["precision"]), list(zip(names, offs, cnts, dts)))
    extra = {k[len("extra/"):]: v for k, v in z.items() if k.startswith("extra/")}
    return snap, extra
