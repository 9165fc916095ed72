"""Reproduce one saved environment (a file written by tools/probe_unstable.py): restore it into a 1-environment handle, replay the saved
actions once, and report whether the same warn bits and the same final state come back.  A per-environment rollout does not depend on the
batch around it, so under the same library build, precision and mode the replay is bit-identical to the original event.
usage: python tools/replay_snapshot.py <snapshot.npz>   (exit status 0: reproduced, 1: not reproduced)"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import robosuite_b200 as suite  # noqa: E402
from robosuite_b200.state_io import load_snapshot  # noqa: E402

snap, extra = load_snapshot(sys.argv[1])
task, robot, acts = str(extra["task"]), str(extra["robot"]), extra["actions"]
env = suite.make(task, robots=robot, num_envs=1, seed=1, horizon=10 ** 9, precision=snap.precision)
tensors = {k: torch.as_tensor(v, device=env.device) for k, v in extra.items()
           if k in ("timestep", "done") + tuple(env._task_state)}
env.set_env_state({"sim": snap, "tensors": tensors, "host_steps": None, "max_steps": int(tensors["timestep"].max())})
for a in acts:
    env.step(torch.as_tensor(a[None], dtype=env.dtype, device=env.device))
torch.cuda.synchronize()
warn = int(env.sim.warn[0])
qpos, qvel = env.sim.qpos[0].cpu().numpy(), env.sim.qvel[0].cpu().numpy()
same_warn = warn == int(extra["warn_after"])
same_state = np.array_equal(qpos, extra["qpos_after"]) and np.array_equal(qvel, extra["qvel_after"], equal_nan=True)
print("%s/%s %s, %d actions replayed: warn %d (saved %d) %s, final qpos / qvel %s" % (
    task, robot, snap.precision, len(acts), warn, int(extra["warn_after"]), "same" if same_warn else "DIFFERENT",
    "bit-identical" if same_state else "DIFFERENT (max |dqpos| %.3g)" % float(np.nanmax(np.abs(qpos - extra["qpos_after"])))))
env.close()
sys.exit(0 if same_warn and same_state else 1)
