"""Where does run-to-run nondeterminism of the pipeline come from?  For each configuration (library switches set through the
environment before the handles are created) run T trials of: two handles stepping concurrently on two streams + one handle alone,
compare all state arrays after every control step, print the first divergence.
usage: python tools/debug_nondet.py [trials] [n_env] [steps]"""
import ctypes as C
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests import test_gpu_boundary as T  # noqa: E402
from tests.util import lift_states, load  # noqa: E402
from robosuite_b200.mjcf.compiler import pack_model  # noqa: E402

L = T._lib()
model = load("Lift_Panda")
blob = pack_model(model)
trials = int(sys.argv[1]) if len(sys.argv) > 1 else 3
n = int(sys.argv[2]) if len(sys.argv) > 2 else 64
steps = int(sys.argv[3]) if len(sys.argv) > 3 else 12
q, _ = lift_states(model, n, seed=31)
rng = np.random.default_rng(4)
acts = rng.uniform(-1, 1, size=(steps, n, 7))
acts[:, : n // 2, 2] = -1.0
acts[:, :, 6] = 1.0
acts_d = torch.as_tensor(acts, dtype=torch.float32, device="cuda")
NAMES = ["qpos", "qvel", "qacc_warmstart", "ctrl", "ctrl_goal_pos", "ctrl_goal_ori", "ctrl_torque", "warn", "time"]
KEYS = ["B2S_GROUPS", "B2S_CTRL_SPLIT", "B2S_NO_GJK_CACHE"]
CONFIGS = [
    ("default", {"B2S_NO_GJK_CACHE": "1"}),
    ("G1", {"B2S_NO_GJK_CACHE": "1", "B2S_GROUPS": "1"}),
    ("nosplit", {"B2S_NO_GJK_CACHE": "1", "B2S_CTRL_SPLIT": "0"}),
    ("G1_nosplit", {"B2S_NO_GJK_CACHE": "1", "B2S_GROUPS": "1", "B2S_CTRL_SPLIT": "0"}),
]
only = os.environ.get("ONLY")


def setup(stream):
    h = T._create(L, blob, n, 0)
    if stream is not None:
        assert L.b2s_set_stream(h, C.c_void_p(stream.cuda_stream)) == 0
    c = T._lift_osc_cfg(L, h)
    assert L.b2s_ctrl_config(h, C.byref(c)) == 0
    assert L.b2s_set_export(h, 0) == 0 and L.b2s_set_mode(h, 1) == 0
    with torch.cuda.stream(stream) if stream is not None else torch.cuda.stream(torch.cuda.current_stream()):
        T._arr(L, h, "qpos").copy_(torch.as_tensor(q, dtype=torch.float32))
        assert L.b2s_forward(h) == 0 and L.b2s_ctrl_reset(h, None) == 0
    return h


for name, envs in CONFIGS:
    if only and name not in only.split(","):
        continue
    for k in KEYS:
        os.environ.pop(k, None)
    os.environ.update(envs)
    res = []
    for trial in range(trials):
        sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
        ha, hb, hc = setup(sa), setup(sb), setup(None)
        torch.cuda.synchronize()
        first = None
        if os.environ.get("NOSYNC"):
            for t in range(steps):
                with torch.cuda.stream(sa):
                    assert L.b2s_env_step(ha, C.c_void_p(acts_d[t].data_ptr()), 25) == 0
                with torch.cuda.stream(sb):
                    assert L.b2s_env_step(hb, C.c_void_p(acts_d[t].data_ptr()), 25) == 0
            torch.cuda.synchronize()
            for t in range(steps):
                assert L.b2s_env_step(hc, C.c_void_p(acts_d[t].data_ptr()), 25) == 0
            torch.cuda.synchronize()
            for nm in NAMES:
                try:
                    a, b, c = (T._arr(L, h, nm) for h in (ha, hb, hc))
                except Exception:
                    continue
                for tag, x, y in (("AB", a, b), ("AC", a, c), ("BC", b, c)):
                    if not torch.equal(x, y):
                        d = (x.double() - y.double()).abs().reshape(n, -1)
                        ev = torch.nonzero(d.amax(1) > 0).flatten().tolist()
                        first = first or []
                        first.append((steps, nm, tag, ev[:8], float(d.max())))
        for t in range(steps if not os.environ.get("NOSYNC") else 0):
            with torch.cuda.stream(sa):
                assert L.b2s_env_step(ha, C.c_void_p(acts_d[t].data_ptr()), 25) == 0
            with torch.cuda.stream(sb):
                assert L.b2s_env_step(hb, C.c_void_p(acts_d[t].data_ptr()), 25) == 0
            torch.cuda.synchronize()
            assert L.b2s_env_step(hc, C.c_void_p(acts_d[t].data_ptr()), 25) == 0
            torch.cuda.synchronize()
            for nm in NAMES:
                try:
                    a, b, c = (T._arr(L, h, nm) for h in (ha, hb, hc))
                except Exception:
                    continue
                for tag, x, y in (("AB", a, b), ("AC", a, c), ("BC", b, c)):
                    if not torch.equal(x, y):
                        d = (x.double() - y.double()).abs().reshape(n, -1)
                        ev = torch.nonzero(d.amax(1) > 0).flatten().tolist()
                        first = first or []
                        first.append((t, nm, tag, ev[:8], float(d.max())))
            if first:
                break
        res.append(first)
        for h in (ha, hb, hc):
            L.b2s_destroy(h)
    nd = sum(1 for r in res if r)
    print(f"[{name}] {nd}/{trials} trials diverged")
    for r in res:
        if r:
            for x in r[:6]:
                print("    step %d %s %s envs %s max|d| %.3g" % x)
            print("    ..")
    sys.stdout.flush()
