"""Cost of whole-environment snapshots on 4096 Lift/Panda environments (f32, pipeline mode): row size, and CUDA-event times of
snapshot-all, restore-all and a random-permutation clone (snapshot-all + restore), each over `reps` repetitions after warm-up, beside the
time of one control step of the same batch measured in the same run.  Prints the card name and power limit with the numbers.
usage: python tools/probe_snapshot.py [n_env] [reps]"""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import robosuite_b200 as suite  # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 200
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                      capture_output=True, text=True).stdout.strip()
env = suite.make("Lift", robots="Panda", num_envs=n, seed=0, horizon=10 ** 9)
sim = env.sim
g = torch.Generator(device=env.device)
g.manual_seed(0)
acts = [torch.rand((n, env.action_dim), generator=g, device=env.device, dtype=env.dtype) * 2 - 1 for _ in range(8)]
perm = torch.randperm(n, generator=g, device=env.device).to(torch.int32)
for a in acts:  # contacts, warm starts and the GJK cache in use
    env.step(a)
snap = sim.snapshot()


def timed(fn, k):
    for _ in range(3):
        fn(0)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for i in range(k):
        fn(i)
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / k


res = {
    "card": card, "n_env": n, "reps": reps, "row_bytes": int(snap.rows.shape[1]), "nsections": len(snap.sections),
    "snapshot_all_ms": timed(lambda i: sim.snapshot(), reps),
    "restore_all_ms": timed(lambda i: sim.restore(snap), reps),
    "clone_permutation_ms": timed(lambda i: sim.clone_envs(perm), reps),
    "control_step_ms": timed(lambda i: env.step(acts[i % len(acts)]), reps),
}
res["snapshot_GB_per_s"] = n * res["row_bytes"] * 2 / (res["snapshot_all_ms"] * 1e-3) / 1e9  # bytes read + written
print(json.dumps(res))
env.close()
