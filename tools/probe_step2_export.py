"""Device time of one Lift/Panda control step (env.step) with and without the step-2 arrays, f32, CUDA events around K steps after W
warm-up steps, random actions.  Configurations, alternated over R rounds so that their spread can be read beside their difference:
  pipeline            the pipeline schedule, no export (the default);
  pipeline+step2      the pipeline with the step-2 export and the contact records (make(dynamics_queries=True));
  pipeline+query      the same plus one sim.data.contact_force() and one sim.data.actuator_force read per step (the query's torch
                      ops on the step's stream);
  fused+full_export   set_export(True): what delivered these arrays before the step-2 export - the fused kernel writing every
                      derived array (poses, qM, contacts, efc rows, actuator forces) on the last substep.
Prints one JSON line per configuration and round, with the card's name and power limit.
usage: python tools/probe_step2_export.py [n_env=4096] [steps=20] [warmup=5] [rounds=3]"""
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
W = int(sys.argv[3]) if len(sys.argv) > 3 else 5
R = int(sys.argv[4]) if len(sys.argv) > 4 else 3
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                   capture_output=True, text=True).stdout.strip().split(", ")

CONFIGS = {
    "pipeline": dict(kw={}, full=False, query=False),
    "pipeline+step2": dict(kw={"dynamics_queries": True}, full=False, query=False),
    "pipeline+query": dict(kw={"dynamics_queries": True}, full=False, query=True),
    "fused+full_export": dict(kw={}, full=True, query=False),
}


def measure(cfg):
    env = suite.make("Lift", robots="Panda", num_envs=n, seed=1, horizon=10 ** 9, precision="f32", **cfg["kw"])
    if cfg["full"]:
        env.sim.set_export(True)
    gen = torch.Generator(device=env.device)
    gen.manual_seed(3)
    acts = torch.rand((W + K, n, env.action_dim), generator=gen, device=env.device, dtype=env.dtype) * 2 - 1
    acc = torch.zeros((n, 6), dtype=env.dtype, device=env.device)

    def step(a):
        env.step(a)
        if cfg["query"]:
            acc.add_(env.sim.data.contact_force().sum(1))
            acc[:, 0].add_(env.sim.data.actuator_force[:, 0])

    for k in range(W):
        step(acts[k])
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for k in range(W, W + K):
        step(acts[k])
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / K
    env.close()
    return ms


for r in range(R):
    for name, cfg in CONFIGS.items():
        ms = measure(cfg)
        print(json.dumps({"config": name, "round": r, "n_env": n, "steps": K, "ms_per_step": round(ms, 3),
                          "env_steps_per_s": round(n * 1000.0 / ms), "gpu": q[0],
                          "power_limit": q[1] if len(q) > 1 else None}), flush=True)
