"""Device time of one Lift/Panda control step (env.step) with and without the contact records, f32, CUDA events around K steps after
W warm-up steps, random actions.  Configurations, alternated over R rounds so that their spread can be read beside their difference:
  pipeline            the pipeline schedule, no export (the default);
  pipeline+contacts   the pipeline with the contact export (make(contact_queries=True));
  pipeline+query      the same plus one env._check_grasp(cube) per step (the query's torch ops on the step's stream);
  unit+contacts       the unit queue (mode 2) with the contact export;
  fused+full_export   set_export(True): what delivered contacts before the contact export - the fused kernel writing every derived
                      array (poses, qM, cdof, efc rows, actuator forces) on the last substep.
Prints one JSON line per configuration and round, with the card's name and power limit.
usage: python tools/probe_contacts.py [n_env=4096] [steps=20] [warmup=5] [rounds=3]"""
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
    "pipeline": dict(kw={}, mode=None, full=False, query=False),
    "pipeline+contacts": dict(kw={"contact_queries": True}, mode=None, full=False, query=False),
    "pipeline+query": dict(kw={"contact_queries": True}, mode=None, full=False, query=True),
    "unit+contacts": dict(kw={"contact_queries": True}, mode=2, full=False, query=False),
    "fused+full_export": dict(kw={}, mode=None, full=True, query=False),
}


def measure(cfg):
    env = suite.make("Lift", robots="Panda", num_envs=n, seed=1, horizon=10 ** 9, precision="f32", **cfg["kw"])
    if cfg["mode"] is not None:
        env.sim.set_mode(cfg["mode"])
    if cfg["full"]:
        env.sim.set_export(True)
    gen = torch.Generator(device=env.device)
    gen.manual_seed(3)
    acts = torch.rand((W + K, n, env.action_dim), generator=gen, device=env.device, dtype=env.dtype) * 2 - 1
    grasped = torch.zeros(n, dtype=torch.long, device=env.device)

    def step(a):
        env.step(a)
        if cfg["query"]:
            grasped.add_(env._check_grasp(env.cube_geoms).long())

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
    ncon = float(env.sim.ncon.float().mean()) if cfg["kw"] or cfg["full"] else None
    env.close()
    return ms, ncon


for r in range(R):
    for name, cfg in CONFIGS.items():
        ms, ncon = measure(cfg)
        print(json.dumps({"config": name, "round": r, "n_env": n, "steps": K, "ms_per_step": round(ms, 3),
                          "env_steps_per_s": round(n * 1000.0 / ms), "mean_ncon_last_substep": ncon, "gpu": q[0],
                          "power_limit": q[1] if len(q) > 1 else None}), flush=True)
