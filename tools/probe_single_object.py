"""Device time of one control step of PickPlace and its single-object variants (env.step: the engine's substeps, the task's reward
and success tensors), CUDA events around K steps after W warm-up steps, random actions, pipeline schedule.  Prints one JSON line per
task with the card's name and power limit beside the numbers.
usage: python tools/probe_single_object.py [n_env=4096] [steps=20] [warmup=10] [task ...]"""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import robosuite_b200 as suite  # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
K = int(sys.argv[2]) if len(sys.argv) > 2 else 20
W = int(sys.argv[3]) if len(sys.argv) > 3 else 10
tasks = sys.argv[4:] or ["PickPlace", "PickPlaceCan", "PickPlaceSingle", "NutAssemblySingle"]
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                   capture_output=True, text=True).stdout.strip().split(", ")
for task in tasks:
    env = suite.make(task, robots="Panda", num_envs=n, seed=1, horizon=10 ** 9)
    gen = torch.Generator(device=env.device)
    gen.manual_seed(3)
    acts = torch.rand((W + K, n, env.action_dim), generator=gen, device=env.device, dtype=env.dtype) * 2 - 1
    for k in range(W):
        env.step(acts[k])
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for k in range(W, W + K):
        env.step(acts[k])
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / K
    print(json.dumps({"task": task, "n_env": n, "steps": K, "ms_per_step": round(ms, 3), "env_steps_per_s": round(n * 1000.0 / ms),
                      "envs_with_warn": int((env.sim.warn != 0).sum()), "tier_small": env.tier_small, "gpu": q[0],
                      "power_limit": q[1] if len(q) > 1 else None}), flush=True)
    env.close()
