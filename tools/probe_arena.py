"""Cost of per-environment tables on the Lift throughput path: 4096 environments stepped with random actions, the table arguments
off (the default table) and on (table_full_size and table_friction as [n_env, 3] arrays), and the time of one set_table + masked
reset of a quarter of the environments.  Prints one JSON line per measurement with the GPU name and power limit they belong to.

    python tools/probe_arena.py [n_env] [steps]
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


def gpu():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, check=True).stdout.strip().splitlines()[0]
    except Exception as e:  # the numbers are only meaningful with the card beside them
        return "unknown (%s)" % e


def make(n, per_env):
    kw = {}
    if per_env:
        r = np.random.default_rng(0)
        kw = dict(table_full_size=np.column_stack([r.uniform(0.6, 1.2, n), r.uniform(0.6, 1.2, n), r.uniform(0.03, 0.1, n)]),
                  table_friction=np.column_stack([r.uniform(0.5, 2.0, n), np.full(n, 5e-3), np.full(n, 1e-4)]))
    return suite.make("Lift", robots="Panda", num_envs=n, seed=1, ignore_done=True, **kw)


def steps_per_s(env, steps):
    g = torch.Generator(device=env.device)
    g.manual_seed(0)
    acts = torch.rand((steps, env.num_envs, env.action_dim), generator=g, device=env.device, dtype=env.dtype) * 2 - 1
    for t in range(20):  # warm-up: graphs captured, every launch shape seen
        env.step(acts[t])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for t in range(steps):
        env.step(acts[t])
    torch.cuda.synchronize()
    return env.num_envs * steps / (time.perf_counter() - t0)


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 200
    card = gpu()
    for per_env in (False, True, False, True):  # alternating: the spread of each setting shows beside the difference
        env = make(n, per_env)
        print(json.dumps({"probe": "arena", "n_env": n, "per_env_table": per_env, "env_steps_per_s": round(steps_per_s(env, steps)),
                          "gpu": card}), flush=True)
        if per_env:
            mask = torch.zeros(n, dtype=torch.bool, device=env.device)
            mask[::4] = True
            for k in range(3):  # the first call includes one-time set-up
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                env.set_table(full_size=(1.0, 0.8, 0.06), friction=(1.5, 5e-3, 1e-4), mask=mask)
                env.reset(mask=mask)
                torch.cuda.synchronize()
                ms = (time.perf_counter() - t0) * 1e3
            print(json.dumps({"probe": "arena_set_table_reset", "n_env": n, "masked": int(mask.sum()), "ms": round(ms, 3), "gpu": card}),
                  flush=True)
        env.close()


if __name__ == "__main__":
    main()
