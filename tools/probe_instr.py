"""Device timeline + solver statistics of one control step in steady state (needs a -DB2S_INSTR build of the library:
B2S_LIB=robosuite_b200/variants/libb2s_instr.so).  Answers, from data of the CUDA-graph replay itself:
  * how long each kernel of a group-substep runs and how long the gaps between dependent kernels are (%globaltimer stamps);
  * the Newton-iteration / ncon / nefc histograms and line-search evaluations per solve;
  * how unevenly the environments of one block cost (clock64 per environment-substep): block time = slowest warp.  Tail blocks are
    the ones the environments were recorded running in; phase-0 blocks are taken as 8 consecutive warps, the launch bounds' cap and
    what the Lift / Panda f32 layout gets (for models whose phase-0 blocks hold fewer warps that grouping is approximate).
usage: python tools/probe_instr.py [task] [robot] [n_env] [controller] -> JSON on stdout"""
import json
import os
import sys

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import robosuite_b200 as suite  # noqa: E402
from robosuite_b200 import controller_config as cc  # noqa: E402

task = sys.argv[1] if len(sys.argv) > 1 else "Lift"
robot = sys.argv[2] if len(sys.argv) > 2 else "Panda"
n = int(sys.argv[3]) if len(sys.argv) > 3 else 4096
ctrl = sys.argv[4] if len(sys.argv) > 4 else "OSC_POSE"
kw = {}
if ctrl != "OSC_POSE":
    kw["controller_configs"] = cc.refactor_composite_controller_config(cc.load_part_controller_config(ctrl), robot, ["right"])
env = suite.make(task, robots=robot, num_envs=n, seed=1, horizon=10 ** 9, **kw)
sim = env.sim
gen = torch.Generator(device=env.device)
gen.manual_seed(3)
for i in range(int(os.environ.get("PREROLL", "100"))):
    sim.env_step(torch.rand((n, env.action_dim), generator=gen, device=env.device, dtype=env.dtype) * 2 - 1, 25)
torch.cuda.synchronize()
sim.stats.zero_()
act = torch.rand((n, env.action_dim), generator=gen, device=env.device, dtype=env.dtype) * 2 - 1
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
sim.env_step(act, 25)
e1.record()
torch.cuda.synchronize()
step_ms = e0.elapsed_time(e1)
b = sim.st_begin.cpu().numpy().astype(np.uint64).reshape(64, 32, 8)
e = sim.st_end.cpu().numpy().astype(np.uint64).reshape(64, 32, 8)
G = int(os.environ.get("B2S_GROUPS", "8"))
valid = e[:G, :25] > 0
t0 = b[:G, :25][valid].min()
B = (b[:G, :25].astype(np.float64) - float(t0)) / 1e3  # us
E = (e[:G, :25].astype(np.float64) - float(t0)) / 1e3
names = ["P0", "narrowA", "narrowG", "tail", "ctrl"]  # the tail launch runs both capacity tiers
out = {"task": task, "robot": robot, "n_env": n, "controller": ctrl, "groups": G, "step_ms_events": step_ms,
       "span_us": float(E.max()), "kernels": {}, "gaps_us": {}}
for k, nm in enumerate(names):
    if not (e[:G, :25, k] > 0).any():
        continue
    d = E[:, :, k] - B[:, :, k]
    out["kernels"][nm] = {"mean_us": float(d.mean()), "p50": float(np.median(d)), "max": float(d.max()), "sum_per_group_us": float(d.sum(1).mean())}
# gaps between dependent launches of one group: end(prev) -> begin(next)
out["gaps_us"]["P0->narrowA"] = float((B[:, :, 1] - E[:, :, 0]).mean())
out["gaps_us"]["narrowA->narrowG"] = float((B[:, :, 2] - E[:, :, 1]).mean())
out["gaps_us"]["narrowG->tail"] = float((B[:, :, 3] - E[:, :, 2]).mean())
out["gaps_us"]["tail->next P0"] = float((B[:, 1:, 0] - E[:, :-1, 3]).mean())
if "ctrl" in out["kernels"]:
    out["gaps_us"]["P0->ctrl"] = float((B[:, :, 4] - E[:, :, 0]).mean())
    out["gaps_us"]["ctrl->tail"] = float((B[:, :, 3] - E[:, :, 4]).mean())
# a group's serial chain per substep: end of its tail launch of substep s -> end of its tail launch of substep s + 1
ch = E[:, 1:, 3] - E[:, :-1, 3]
out["chain_us"] = {"mean": float(ch.mean()), "p50": float(np.median(ch)), "max": float(ch.max())}
per_group_busy = sum((E[:, :, k] - B[:, :, k]).sum(1) for k in range(4))
out["per_group_kernel_time_us"] = [float(x) for x in per_group_busy]
out["per_group_span_us"] = [float(E[g].max() - B[g].min()) for g in range(G)]
# concurrency: at how many instants are 0/1/2/.. phase kernels (P0 or tail) of different groups running?
ts = np.linspace(0, E.max(), 4000)
run = np.zeros_like(ts)
for g in range(G):
    for s in range(25):
        for k in (0, 3):
            run += (ts >= B[g, s, k]) & (ts < E[g, s, k])
out["phase_kernels_running_hist"] = {str(i): float((run == i).mean()) for i in range(G + 1)}
st = sim.stats.cpu().numpy()
nsolve = max(int(st[17]), 1)
nc, ne = st[32:161], st[176:497]


def pct(h, q):
    c = np.cumsum(h) / max(h.sum(), 1)
    return int(np.searchsorted(c, q))


out["solver"] = {"solves": int(st[17]), "niter_hist": st[:16].tolist(), "mean_niter": float((st[:16] * np.arange(16)).sum() / max(st[:16].sum(), 1)),
                 "ls_evals_per_solve": float(st[16]) / nsolve, "large_tier_env_substeps": int(st[19]),
                 "ncon": {"mean": float((nc * np.arange(len(nc))).sum() / max(nc.sum(), 1)), "p99": pct(nc, 0.99), "p999": pct(nc, 0.999), "max": int(np.nonzero(nc)[0].max())},
                 "nefc": {"mean": float((ne * np.arange(len(ne))).sum() / max(ne.sum(), 1)), "p99": pct(ne, 0.99), "p999": pct(ne, 0.999), "max": int(np.nonzero(ne)[0].max())},
                 "ncon_hist": nc.tolist(), "nefc_hist": ne.tolist()}
out["convex_items"] = {"hits": int(st[18]), "cycles_log2_bucket0_is_256": {"other": st[488:500].tolist(), "mesh_mesh": st[476:488].tolist()}}
sl = sim.slowlog.cpu().numpy()
gn = env.model.names["geom"]
out["slow_items"] = [dict(cycles=int(r[0]), types=(int(r[1]), int(r[2])), nvert=(int(r[3]), int(r[4])), epa_nV=int(r[5]), epa_nF=int(r[6]), gjk_cycles=int(r[7]),
                          hit=int(r[8]), staged=int(r[9]), geoms=(gn[int(r[10])], gn[int(r[11])])) for r in sl if r[0] > 0][:40]
out["slow_items_total"] = int(st[20])
cy = sim.cyc.cpu().numpy()[:, :25]  # [n, 25, 8]: P0 cycles, tail cycles, ..., tail block index
for k, nm in ((0, "P0"), (1, "tail")):
    c = cy[:, :, k]
    ratios, lratios = [], []
    for g in range(G):
        e0, e1 = n * g // G, n * (g + 1) // G
        cg = c[e0:e1]
        # phase 0: environment env0 + 8 b + w runs in block b; the tail records the block each environment-substep ran in
        bg = cy[e0:e1, :, 7].astype(np.int64) if k == 1 else np.repeat((np.arange(e1 - e0) // 8)[:, None], 25, 1)
        for s in range(25):
            cnt = np.bincount(bg[:, s])
            mx = np.zeros(len(cnt))
            np.maximum.at(mx, bg[:, s], cg[:, s])
            ok = cnt > 0
            ratios.append(float((mx[ok] / np.maximum(np.bincount(bg[:, s], cg[:, s])[ok] / cnt[ok], 1)).mean()))  # block time / mean warp time
        lratios.append(float((cg.max(0) / np.maximum(cg.mean(0), 1)).mean()))    # launch time / mean warp time
    out["cycles_" + nm] = {"mean": float(c.mean()), "p50": float(np.median(c)), "p90": float(np.percentile(c, 90)),
                           "p99": float(np.percentile(c, 99)), "max": float(c.max()),
                           "block_max_over_mean": float(np.mean(ratios)), "launch_max_over_mean": float(np.mean(lratios))}
out["warn"] = int(sim.warn.abs().max())
out["raw_begin_us"] = np.where(e[:G, :25] > 0, B, -1).round(1).tolist()  # [group][substep][kind]
out["raw_end_us"] = np.where(e[:G, :25] > 0, E, -1).round(1).tolist()
print(json.dumps(out))
