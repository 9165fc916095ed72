"""How much of the tail kernel's block slack an environment order could recover, from one control step of the -DB2S_INSTR build
(B2S_LIB=robosuite_b200/variants/libb2s_instr.so) in steady state.

A tail block holds an SM until its slowest warp is done, so a block costs the maximum of its environments' tail cycles and the launch's
SM-time is the sum of those maxima.  From the recorded cost and counts of every environment-substep (`cyc`) this computes, per order
of each group's environments:
  * the mean over blocks of block max / block mean and the summed block maxima (relative to the order the blocks really ran in);
  * for the orders sorted by a key of the PREVIOUS substep, how much of the gap between the order that ran and the true-cost order
    (the bound: sorted by this substep's own cost) they recover.
Orders: "ran" (the blocks the environments really ran in), "by_id" (consecutive environment ids), "prev_<key>" (most expensive key of
the previous substep first), "true" (this substep's cost).  Keys: the previous substep's cycles, Newton iterations, line-search
evaluations, nefc, ncon, a least-squares cost model of those counts, and `bucket`, the tail's cost class (tail_cost_key in
b2s_pipeline.cuh).  The cycles are taken with the co-residency of the order that ran, so the sorted orders' figures are estimates.
usage: python tools/probe_tail_order.py [task] [robot] [n_env] -> JSON on stdout"""
import json
import os
import sys

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import robosuite_b200 as suite  # noqa: E402

task = sys.argv[1] if len(sys.argv) > 1 else "Lift"
robot = sys.argv[2] if len(sys.argv) > 2 else "Panda"
n = int(sys.argv[3]) if len(sys.argv) > 3 else 4096
NSUB = 25
env = suite.make(task, robots=robot, num_envs=n, seed=1, horizon=10 ** 9)
sim = env.sim
gen = torch.Generator(device=env.device)
gen.manual_seed(3)
for i in range(int(os.environ.get("PREROLL", "100"))):
    sim.env_step(torch.rand((n, env.action_dim), generator=gen, device=env.device, dtype=env.dtype) * 2 - 1, NSUB)
torch.cuda.synchronize()
if not hasattr(sim, "cyc"):
    sys.exit("probe_tail_order.py needs the -DB2S_INSTR library: B2S_LIB=robosuite_b200/variants/libb2s_instr.so")
sim.env_step(torch.rand((n, env.action_dim), generator=gen, device=env.device, dtype=env.dtype) * 2 - 1, NSUB)
torch.cuda.synchronize()
cy = sim.cyc.cpu().numpy()[:, :NSUB].astype(np.float64)  # [n, substep, 8]
cost, niter, ls, nefc, ncon, large, blk = (cy[:, :, k] for k in range(1, 8))
G = int(os.environ.get("B2S_GROUPS", "8"))
bounds = [(n * g // G, n * (g + 1) // G) for g in range(G)]


def bucket(niter, nefc, large):
    """tail_cost_key of b2s_pipeline.cuh, on the recorded counts"""
    w = niter * (nefc + 24) + 2 * nefc
    return np.where(large > 0, 15, np.minimum(14, w // 48))


# least-squares cost model of the counts (fitted on this run): what a key built from the counts could predict at best
X = np.stack([np.ones_like(cost), nefc, ncon, niter, niter * nefc, ls, ls * nefc, large], -1).reshape(-1, 8)
coef = np.linalg.lstsq(X, cost.reshape(-1), rcond=None)[0]
model = (X @ coef).reshape(cost.shape)
keys = {"cycles": cost, "niter": niter, "ls": ls, "nefc": nefc, "ncon": ncon, "model": model, "bucket": bucket(niter, nefc, large)}
ran_blocks = [int(blk[e0:e1].max()) + 1 for e0, e1 in bounds]
wpb = int(max(np.bincount(blk[e0:e1, 0].astype(np.int64)).max() for e0, e1 in bounds))


def blocks_of(order_cost):
    """order_cost: [nenv] costs in warp-position order -> per-block max and mean"""
    nb = (len(order_cost) + wpb - 1) // wpb
    pad = np.full(nb * wpb, np.nan)
    pad[:len(order_cost)] = order_cost
    b = pad.reshape(nb, wpb)
    return np.nanmax(b, 1), np.nanmean(b, 1)


def score(order_fn):
    """mean block max / mean and summed block maxima over groups and substeps 1..NSUB-1"""
    ratios, summax = [], 0.0
    for e0, e1 in bounds:
        for s in range(1, NSUB):
            c = cost[e0:e1, s]
            mx, mn = blocks_of(c[order_fn(e0, e1, s)])
            ratios.append((mx / np.maximum(mn, 1)).mean())
            summax += mx.sum()
    return float(np.mean(ratios)), summax


def by_key(k):
    # most expensive first; ties keep the id order
    return lambda e0, e1, s: np.argsort(-k[e0:e1, s - 1], kind="stable")


out = {"task": task, "robot": robot, "n_env": n, "groups": G, "warps_per_tail_block": wpb, "orders": {}}
# the blocks the environments really ran in (recorded block index per environment-substep)
ratios, lratios, summax = [], [], 0.0
for e0, e1 in bounds:
    for s in range(1, NSUB):
        c, b = cost[e0:e1, s], blk[e0:e1, s].astype(np.int64)
        mx = np.zeros(b.max() + 1)
        np.maximum.at(mx, b, c)
        mn = np.bincount(b, c) / np.maximum(np.bincount(b), 1)
        ok = np.bincount(b) > 0
        ratios.append((mx[ok] / np.maximum(mn[ok], 1)).mean())
        lratios.append(c.max() / max(c.mean(), 1))
        summax += mx[ok].sum()
ref = summax
out["orders"]["ran"] = {"block_max_over_mean": float(np.mean(ratios)), "launch_max_over_mean": float(np.mean(lratios)), "sum_block_max_rel": 1.0}
orders = {"by_id": lambda e0, e1, s: np.arange(e1 - e0), "true": lambda e0, e1, s: np.argsort(-cost[e0:e1, s], kind="stable")}
orders.update({"prev_" + k: by_key(v) for k, v in keys.items()})
res = {k: score(f) for k, f in orders.items()}
for k, (r, sm) in res.items():
    out["orders"][k] = {"block_max_over_mean": r, "sum_block_max_rel": sm / ref}
gap = ref - res["true"][1]
for k in keys:
    out["orders"]["prev_" + k]["recovered_of_gap"] = float((ref - res["prev_" + k][1]) / gap) if gap > 0 else 0.0
# how well the previous substep's key predicts this substep's cost
out["corr_with_next_cost"] = {k: float(np.corrcoef(v[:, :-1].ravel(), cost[:, 1:].ravel())[0, 1]) for k, v in keys.items()}
out["corr_with_same_cost"] = {k: float(np.corrcoef(v.ravel(), cost.ravel())[0, 1]) for k, v in keys.items()}
out["cost_model_coef"] = dict(zip(["1", "nefc", "ncon", "niter", "niter*nefc", "ls", "ls*nefc", "large"], coef.round(1).tolist()))
bk = keys["bucket"]
out["bucket"] = {"count": np.bincount(bk.astype(np.int64).ravel(), minlength=16).tolist(),
                 "mean_cycles": [float(cost[bk == k].mean()) if (bk == k).any() else 0.0 for k in range(16)]}
out["cycles"] = {"mean": float(cost.mean()), "p50": float(np.median(cost)), "p90": float(np.percentile(cost, 90)),
                 "p99": float(np.percentile(cost, 99)), "max": float(cost.max())}
out["counts"] = {"niter_hist": np.bincount(niter.astype(np.int64).ravel()).tolist(), "nefc_p50_p90_p99_max": np.percentile(nefc, [50, 90, 99, 100]).tolist(),
                 "w_p10_p50_p90_p99_max": np.percentile(niter * (nefc + 24) + 2 * nefc, [10, 50, 90, 99, 100]).tolist(),
                 "large_tier_env_substeps": int(large.sum()), "tail_blocks_per_group": ran_blocks}
print(json.dumps(out))
