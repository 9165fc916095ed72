"""Golden vectors for the environment layer from the REFERENCE'S OWN Python code.

Runs the unmodified robosuite stack (checkout in ROBOSUITE_REFERENCE) on the CPU oracle through oracle/mujoco_shim (a `mujoco`
look-alike) and records, per task: the composed model's reset state, the action sequence, and after every control step
the reference's flat observation (`object-state`, `robot0_proprio-state`), reward, and qpos.  tests/test_gpu_env.py replays
the same states and actions through robosuite_b200 and compares observation layout / values and rewards with what the
reference code produced.  Needs that checkout; output: tests/golden/env_golden.npz

Usage: python tools/gen_env_golden.py
"""
import os, sys, types
from unittest.mock import MagicMock

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
REF = os.environ.get("ROBOSUITE_REFERENCE", "")  # source checkout of the reference robosuite


def install():
    sys.path.insert(0, os.path.join(ROOT, "oracle", "mujoco_shim"))
    sys.path.insert(0, ROOT)
    tc = types.ModuleType("termcolor")
    tc.colored = lambda s, *a, **k: s
    sys.modules["termcolor"] = tc
    for m in ["mujoco.viewer", "qpsolvers", "pynput", "pynput.keyboard", "hid", "mink", "h5py", "gymnasium",
              "gymnasium.spaces", "gymnasium.core"]:
        sys.modules[m] = MagicMock()
    os.environ["NUMBA_DISABLE_JIT"] = "1"
    sys.path.insert(0, REF)


def run(task, robot, steps=6, seed=0, controller=None, **kw):
    import robosuite as suite

    if controller is not None:  # the way demos/demo_control.py:99-103 selects a part controller
        from robosuite.controllers.composite.composite_controller_factory import refactor_composite_controller_config

        part = suite.load_part_controller_config(default_controller=controller)
        kw["controller_configs"] = refactor_composite_controller_config(part, robot, ["right", "left"])

    env = suite.make(task, robots=robot, has_renderer=False, has_offscreen_renderer=False, use_camera_obs=False,
                     hard_reset=False, reward_shaping=True, control_freq=20, seed=seed, **kw)
    obs = env.reset()
    rng = np.random.default_rng(seed + 1)
    low, high = env.action_spec
    rec = {"qpos0": np.array(env.sim.data.qpos), "keys": [k for k in obs.keys()],
           "obs0_object": np.array(obs["object-state"]), "obs0_proprio": np.array(obs["robot0_proprio-state"]),
           "body_pos": np.array(env.sim.model.body_pos), "body_quat": np.array(env.sim.model.body_quat)}
    acts, objs, pros, rews, qs = [], [], [], [], []
    for t in range(steps):
        a = rng.uniform(low, high)
        obs, r, done, info = env.step(a)
        acts.append(a); objs.append(np.array(obs["object-state"])); pros.append(np.array(obs["robot0_proprio-state"]))
        rews.append(r); qs.append(np.array(env.sim.data.qpos))
    rec.update(actions=np.array(acts), obs_object=np.array(objs), obs_proprio=np.array(pros), reward=np.array(rews), qpos=np.array(qs))
    return rec


if __name__ == "__main__":
    install()
    out = {}
    for task, robot in [("Lift", "Panda"), ("Door", "Panda"), ("NutAssemblyRound", "Panda"), ("PickPlace", "Panda"), ("Stack", "Panda"),
                        ("Lift", "Sawyer"), ("Stack", "Sawyer")]:
        rec = run(task, robot)
        for k, v in rec.items():
            out[f"{task}/{k}" if robot == "Panda" else f"{task}_{robot}/{k}"] = np.array(v)
        print(task, "object-state", rec["obs_object"].shape, "proprio", rec["obs_proprio"].shape, "reward", np.round(rec["reward"], 4))
    for ctrl in ("JOINT_POSITION", "JOINT_TORQUE", "OSC_POSITION"):
        rec = run("Lift", "Panda", controller=ctrl)
        for k, v in rec.items():
            out[f"Lift_{ctrl}/{k}"] = np.array(v)
        print("Lift", ctrl, "reward", np.round(rec["reward"], 4))
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "env_golden.npz"), **out)
