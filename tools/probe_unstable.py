"""Catch the first environments that raise engine flags (or exceed a velocity bound) in a long random-action rollout and save what is needed to
replay them: a full environment snapshot (engine rows, episode clock, task tensors) K control steps before the event and the actions in between.
usage: python tools/probe_unstable.py Task [robot] [n_env] [steps] [precision] [out_dir]
  -> <out_dir>/unstable_<Task>_<precision>.npz (summary: qpos, qvel, qacc_warmstart, ctrl, ctrl_goal_* decoded from the snapshots, for the
     CPU oracle) and <out_dir>/unstable_<Task>_<precision>_<i>.npz per event (state_io.save_snapshot; tools/replay_snapshot.py replays it).
     out_dir defaults to <temporary directory>/b2s_unstable."""
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import robosuite_b200 as suite  # noqa: E402
from robosuite_b200.engine import Snapshot  # noqa: E402
from robosuite_b200.state_io import save_snapshot  # noqa: E402

task = sys.argv[1] if len(sys.argv) > 1 else "PickPlace"
robot = sys.argv[2] if len(sys.argv) > 2 else "Panda"
n = int(sys.argv[3]) if len(sys.argv) > 3 else 1024
steps = int(sys.argv[4]) if len(sys.argv) > 4 else 300
prec = sys.argv[5] if len(sys.argv) > 5 else "f32"
K = 6
out = sys.argv[6] if len(sys.argv) > 6 else os.path.join(tempfile.gettempdir(), "b2s_unstable")
os.makedirs(out, exist_ok=True)
env = suite.make(task, robots=robot, num_envs=n, seed=1, horizon=10 ** 9, precision=prec)
sim = env.sim
env.reset()
g = torch.Generator(device=env.device)
g.manual_seed(0)
hist = []  # (environment state before the step, action)
caught, seen = [], torch.zeros(n, dtype=torch.bool, device=env.device)
for t in range(steps):
    a = torch.rand((n, env.action_dim), generator=g, device=env.device, dtype=env.dtype) * 2 - 1
    hist.append((env.get_env_state(), a.clone()))
    hist = hist[-K:]
    env.step(a)
    vmax = sim.qvel.abs().nan_to_num(1e9).amax(1)
    bad = ((sim.warn != 0) | (vmax > 60)) & ~seen
    if bool(bad.any()):
        for e in torch.nonzero(bad).flatten().tolist()[:8]:
            st0 = hist[0][0]
            snap = Snapshot(st0["sim"].rows[e:e + 1], st0["sim"].signature, st0["sim"].precision, st0["sim"].sections)
            acts = torch.stack([h[1][e] for h in hist]).cpu().numpy()
            extra = {k: v[e:e + 1] for k, v in st0["tensors"].items()}
            extra.update(task=np.array(task), robot=np.array(robot), actions=acts, warn_after=np.array(int(sim.warn[e])),
                         qpos_after=sim.qpos[e].cpu().numpy(), qvel_after=sim.qvel[e].cpu().numpy())
            save_snapshot(os.path.join(out, f"unstable_{task}_{prec}_{len(caught)}.npz"), snap, extra=extra)
            field = {k: torch.stack([h[0]["sim"].field(k)[e] for h in hist]).cpu().numpy()
                     for k in ("qpos", "qvel", "qacc_warmstart", "ctrl", "ctrl_goal_pos", "ctrl_goal_ori")}
            caught.append(dict(env=e, t=t, warn=int(sim.warn[e]), vmax=float(vmax[e]), qpos=field["qpos"], qvel=field["qvel"],
                               ws=field["qacc_warmstart"], ctrl=field["ctrl"], gp=field["ctrl_goal_pos"],
                               go=field["ctrl_goal_ori"], act=acts, ncon=int(sim.ncon[e]), nefc=int(sim.nefc[e]),
                               qpos_after=sim.qpos[e].cpu().numpy(), qvel_after=sim.qvel[e].cpu().numpy()))
            print("t", t, "env", e, "warn", int(sim.warn[e]), "vmax %.1f" % float(vmax[e]), flush=True)
        seen |= bad
    if len(caught) >= 24:
        break
print("steps", t + 1, "envs flagged", int(seen.sum()), "of", n, "-> files in", out)
np.savez_compressed(os.path.join(out, f"unstable_{task}_{prec}.npz"), n=len(caught),
                    **{f"{i}/{k}": np.asarray(v) for i, c in enumerate(caught) for k, v in c.items()})
