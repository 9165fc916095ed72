"""Device time of object placement at 4096 environments (CUDA events over many calls after warm-up), one JSON line per case:
- reset: env.reset(mask) with half of the environments masked, the task's default placement against a user sampler with the
  reference's default ranges (Lift, Stack, NutAssemblyRound);
- kernel: b2s_place_objects alone, for those samplers and for a near-infeasible one that runs all 5000 tries of an object in every
  environment (the bound of the kernel's time);
- gym_step: BatchedGymWrapper.step with an auto-reset of 1/8 of the environments in every step, default placement vs sampler.
The first line names the card and its power limit.  Usage: python tools/probe_placement.py [--n 4096] [--iters 200]"""
import argparse
import json
import math
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import robosuite_b200 as suite  # noqa: E402
from robosuite_b200.placement_samplers import SequentialCompositeSampler, UniformRandomSampler  # noqa: E402


def default_sampler(task):
    """the reference's default sampler of each task (lift.py, stack.py, nut_assembly.py _load_model; recalled)"""
    if task == "NutAssemblyRound":
        c = SequentialCompositeSampler("ObjectSampler")
        for name, yr in (("SquareNut", (0.11, 0.225)), ("RoundNut", (-0.225, -0.11))):
            c.append_sampler(UniformRandomSampler(name + "Sampler", mujoco_objects=name, x_range=(-0.115, -0.11), y_range=yr, rotation=None,
                                                  ensure_object_boundary_in_range=False, ensure_valid_placement=True,
                                                  reference_pos=(0, 0, 0.82), z_offset=0.02))
        return c
    h = 0.03 if task == "Lift" else 0.08
    return UniformRandomSampler("ObjectSampler", x_range=(-h, h), y_range=(-h, h), rotation=None, ensure_object_boundary_in_range=False,
                                ensure_valid_placement=True, reference_pos=(0, 0, 0.8), z_offset=0.01)


def infeasible_sampler():
    """cube B can never clear cube A: every environment runs all 5000 of its tries (and gets warn bit 1024)"""
    return UniformRandomSampler("Tight", x_range=(0, 0.001), y_range=(0, 0.001), ensure_object_boundary_in_range=False,
                                reference_pos=(0, 0, 0.8), z_offset=0.01)


def timed(fn, iters, warm=10):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / iters  # us per call


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=4096)
    ap.add_argument("--iters", type=int, default=200)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("probe_placement needs a CUDA device")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps({"gpu": smi.stdout.strip()}))
    n = args.n
    half = torch.zeros(n, dtype=torch.bool, device="cuda")
    half[::2] = True
    for task in ("Lift", "Stack", "NutAssemblyRound"):
        for which in ("default", "sampler"):
            env = suite.make(task, robots="Panda", num_envs=n, seed=0,
                             placement_initializer=default_sampler(task) if which == "sampler" else None)
            us = timed(lambda: env.reset(mask=half), args.iters)
            rec = {"case": "reset", "task": task, "placement": which, "n_env": n, "us_per_reset": round(us, 1)}
            if which == "sampler":
                q = torch.zeros((n, env.model.nq), dtype=torch.float64, device="cuda")
                m8 = half.to(torch.uint8)
                rec["kernel_us"] = round(timed(lambda: env.sim.place_objects(q, m8, 1, 0), args.iters), 1)
            print(json.dumps(rec))
            env.close()
    env = suite.make("Stack", robots="Panda", num_envs=n, seed=0, placement_initializer=infeasible_sampler())
    q = torch.zeros((n, env.model.nq), dtype=torch.float64, device="cuda")
    us = timed(lambda: env.sim.place_objects(q, None, 1, 0), max(args.iters // 10, 5), warm=3)
    torch.cuda.synchronize()
    print(json.dumps({"case": "kernel", "task": "Stack", "placement": "infeasible (all 5000 tries)", "n_env": n, "kernel_us": round(us, 1),
                      "warn_1024_envs": int((env.sim.warn == 1024).sum())}))
    env.close()
    from robosuite_b200.wrappers import BatchedGymWrapper

    H = 8
    for which in ("default", "sampler"):
        env = suite.make("Lift", robots="Panda", num_envs=n, seed=0, horizon=H,
                         placement_initializer=default_sampler("Lift") if which == "sampler" else None)
        w = BatchedGymWrapper(env)
        w.reset()
        env.set_episode_steps(np.arange(n) % H)
        act = torch.zeros((n, env.action_dim), device="cuda", dtype=env.dtype)
        us = timed(lambda: w.step(act), args.iters, warm=2 * H)
        print(json.dumps({"case": "gym_step", "task": "Lift", "placement": which, "n_env": n, "reset_fraction": 1 / H,
                          "us_per_step": round(us, 1)}))
        env.close()


if __name__ == "__main__":
    main()
