"""Device cost of observable sampling rates and corruptors (BatchedMujocoEnv.modify_observable).

4096 Lift/Panda environments, OSC_POSE, fp32, the phase-kernel pipeline; control steps timed with CUDA events after a warm-up, in
four cases: no modifiers, a Gaussian corruptor on every observable, every observable at 40 Hz (two samples per control step, one in
the middle), every observable at 500 Hz (a sample after every substep).  Cases alternate over `--rounds` rounds; the median per case
is reported with the card's name and power limit.

    python tools/probe_obs_modifiers.py [--n 4096] [--steps 50] [--rounds 3] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

CASES = ("none", "gaussian_all", "all_40hz", "all_500hz")


def configure(env, case):
    from robosuite_b200.observables import create_gaussian_noise_corruptor

    for name in env._obs_slices:
        if case == "gaussian_all":
            env.modify_observable(name, "corruptor", create_gaussian_noise_corruptor(0.0, 0.01))
        elif case == "all_40hz":
            env.modify_observable(name, "sampling_rate", 40)
        elif case == "all_500hz":
            env.modify_observable(name, "sampling_rate", 500)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
        return [s.strip() for s in q.split(",")]
    except Exception as e:  # the numbers stay valid; the card is then unknown
        return ["unknown (%s)" % e, "unknown"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch

    import robosuite_b200 as suite

    envs = {}
    for c in CASES:
        env = suite.make("Lift", robots="Panda", num_envs=a.n, seed=0)
        configure(env, c)
        env.reset()
        envs[c] = env
    gen = torch.Generator(device="cuda")
    gen.manual_seed(0)
    acts = torch.rand((a.steps, a.n, envs["none"].action_dim), generator=gen, device="cuda") * 2 - 1
    times = {c: [] for c in CASES}
    for c in CASES:  # warm-up: graph capture, first launches
        for k in range(a.warmup):
            envs[c].sim.env_step(acts[k], 25)
    torch.cuda.synchronize()
    for _ in range(a.rounds):
        for c in CASES:
            sim = envs[c].sim
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for k in range(a.steps):
                sim.env_step(acts[k], 25)
            t1.record()
            torch.cuda.synchronize()
            times[c].append(t0.elapsed_time(t1) / a.steps)
    name, power = card()
    med = {c: sorted(v)[len(v) // 2] for c, v in times.items()}
    res = {"card": name, "power_limit": power, "n_env": a.n, "steps": a.steps, "rounds": a.rounds,
           "ms_per_control_step": med, "all_ms": times,
           "env_steps_per_s": {c: a.n / (ms * 1e-3) for c, ms in med.items()},
           "cost_vs_none": {c: med[c] / med["none"] - 1.0 for c in CASES}}
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "probe_obs_modifiers.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
