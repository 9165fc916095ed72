"""Cost of per-environment cube sizes on the Lift throughput path: 4096 environments, horizon-500 episodes at staggered phases
auto-reset inside BatchedGymWrapper.step with hard_reset=True, BatchedLift(per_env_cube_size) off and on.  Prints one JSON line per
setting (device-timed and end-to-end env-steps/s) and the time of one set-constants launch over all environments, plus the GPU
name and power limit the numbers belong to.

    python tools/probe_model_override.py [n_env] [steps]
"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import robosuite_b200 as suite  # noqa: E402
from robosuite_b200.wrappers import BatchedGymWrapper  # noqa: E402


def gpu():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, check=True).stdout.strip().splitlines()[0]
    except Exception as e:  # the numbers are only meaningful with the card beside them
        return "unknown (%s)" % e


def run(n, steps, per_env):
    env = suite.make("Lift", robots="Panda", num_envs=n, seed=1, horizon=500, hard_reset=True, per_env_cube_size=per_env)
    w = BatchedGymWrapper(env)
    w.reset()
    env.set_episode_steps(np.arange(n) % env.horizon)  # every step resets ~n / 500 environments
    g = torch.Generator(device=env.device)
    g.manual_seed(0)
    acts = torch.rand((steps, n, env.action_dim), generator=g, device=env.device, dtype=env.dtype) * 2 - 1
    for t in range(20):  # warm-up: graphs captured, every launch shape seen
        w.step(acts[t])
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    ev0.record()
    for t in range(steps):
        w.step(acts[t])
    ev1.record()
    torch.cuda.synchronize()
    e2e = time.perf_counter() - t0
    dev = ev0.elapsed_time(ev1) / 1e3
    out = {"per_env_cube_size": per_env, "n_env": n, "steps": steps, "device_env_steps_per_s": n * steps / dev,
           "e2e_env_steps_per_s": n * steps / e2e}
    if per_env:
        for _ in range(3):
            env.sim.set_const()
        torch.cuda.synchronize()
        reps = 20
        ev0.record()
        for _ in range(reps):
            env.sim.set_const()
        ev1.record()
        torch.cuda.synchronize()
        out["set_const_all_envs_ms"] = ev0.elapsed_time(ev1) / reps
        out["sim_warn_max"] = int(env.sim.warn.max())
    env.close()
    return out


if __name__ == "__main__":
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 200
    print(json.dumps({"gpu": gpu()}), flush=True)
    for per_env in (False, True, False, True):
        print(json.dumps(run(n, steps, per_env)), flush=True)
