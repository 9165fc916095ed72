"""Device time of one Lift/Panda control step (env.step) with the OSC_POSE arm in impedance_mode "fixed", "variable_kp" and
"variable", f32, in the pipeline (mode 1) and the unit queue (mode 2); CUDA events around K steps after W warm-up steps.  The
actions are uniform draws from each configuration's action_spec, so the variable modes set gains across their whole range.  The
configurations are alternated over R rounds so that their spread can be read beside their difference.
Prints one JSON line per configuration and round, with the card's name and power limit.
usage: python tools/probe_variable_impedance.py [n_env=4096] [steps=20] [warmup=5] [rounds=3]"""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import robosuite_b200 as suite  # noqa: E402
from robosuite_b200 import controller_config as cc  # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
K = int(sys.argv[2]) if len(sys.argv) > 2 else 20
W = int(sys.argv[3]) if len(sys.argv) > 3 else 5
R = int(sys.argv[4]) if len(sys.argv) > 4 else 3
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                   capture_output=True, text=True).stdout.strip().split(", ")


def measure(impedance, mode):
    arm = cc.load_part_controller_config("OSC_POSE")
    arm["impedance_mode"] = impedance
    env = suite.make("Lift", robots="Panda", num_envs=n, seed=1, horizon=10 ** 9, precision="f32",
                     controller_configs=cc.refactor_composite_controller_config(arm, "Panda", ["right"]))
    env.sim.set_mode(mode)
    low, high = (torch.as_tensor(b, dtype=env.dtype, device=env.device) for b in env.action_spec)
    gen = torch.Generator(device=env.device)
    gen.manual_seed(3)
    acts = low + (high - low) * torch.rand((W + K, n, env.action_dim), generator=gen, device=env.device, dtype=env.dtype)
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
    env.close()
    return ms


for r in range(R):
    for mode, sched in ((1, "pipeline"), (2, "unit")):
        for impedance in ("fixed", "variable_kp", "variable"):
            ms = measure(impedance, mode)
            print(json.dumps({"config": "%s+%s" % (sched, impedance), "round": r, "n_env": n, "steps": K, "ms_per_step": round(ms, 3),
                              "env_steps_per_s": round(n * 1000.0 / ms), "gpu": q[0], "power_limit": q[1] if len(q) > 1 else None}),
                  flush=True)
