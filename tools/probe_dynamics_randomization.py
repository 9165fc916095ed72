"""Cost of dynamics randomisation on the Lift throughput path: 4096 environments, horizon-500 episodes at staggered phases
auto-reset inside BatchedGymWrapper.step, (a) without BatchedDomainRandomizationWrapper, (b) randomising at resets only, (c) also
before every step (randomize_every_n_steps=1, the reference's default).  Prints one JSON line per setting (device-timed and end-to-end
env-steps/s) and the time of one perturbation launch over all environments, plus the GPU name and power limit the numbers belong to.

    python tools/probe_dynamics_randomization.py [n_env] [steps]
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
from robosuite_b200.wrappers import BatchedDomainRandomizationWrapper, BatchedGymWrapper  # noqa: E402

SETTINGS = {"none": None, "on_reset": 0, "every_step": 1}  # randomize_every_n_steps (None: no randomisation wrapper)


def gpu():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, check=True).stdout.strip().splitlines()[0]
    except Exception as e:  # the numbers are only meaningful with the card beside them
        return "unknown (%s)" % e


def run(n, steps, setting):
    env = suite.make("Lift", robots="Panda", num_envs=n, seed=1, horizon=500)
    k = SETTINGS[setting]
    inner = env if k is None else BatchedDomainRandomizationWrapper(env, seed=3, randomize_every_n_steps=k)
    w = BatchedGymWrapper(inner)
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
    out = {"setting": setting, "n_env": n, "steps": steps, "device_env_steps_per_s": n * steps / dev,
           "e2e_env_steps_per_s": n * steps / e2e}
    if k is not None:
        out["perturb_entries"] = len(inner.perturb_spec)
        reps = 50
        ev0.record()
        for _ in range(reps):
            inner.randomize_domain()
        ev1.record()
        torch.cuda.synchronize()
        out["perturb_all_envs_ms"] = ev0.elapsed_time(ev1) / reps
        out["sim_warn_max"] = int(env.sim.warn.max())
    env.close()
    return out


if __name__ == "__main__":
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 200
    print(json.dumps({"gpu": gpu()}), flush=True)
    for _ in range(2):
        for setting in SETTINGS:
            print(json.dumps(run(n, steps, setting)), flush=True)
