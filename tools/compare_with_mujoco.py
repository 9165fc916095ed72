"""Compare this repo's physics (CPU oracle, and the CUDA engine when a GPU is present) with REAL MuJoCo on the task models.

The build container and the GPU box have no `mujoco` wheel, so the oracle is pinned through the reference's own Python stack on
`oracle/mujoco_shim` (tests/golden/*) - this script is the missing direct check for a machine that has `pip install mujoco`
(any 3.x; the reference pins mujoco>=3.3.0, /root/reference/setup.py:27-39) and the robosuite asset directory:

    python tools/compare_with_mujoco.py --assets $(python -c "import robosuite,os;print(os.path.dirname(robosuite.__file__))")/models/assets
    python tools/compare_with_mujoco.py --assets ... --tasks Lift_Panda Stack_Panda --steps 500 --device

What it does, per task model (tests/golden/mjcf/<task>.xml, composed by the reference's own model composer):
  1. loads the MJCF into mujoco.MjModel (asset paths rewritten to --assets, textures dropped: they do not affect the dynamics) and
     compares the COMPILED constants with robosuite_b200.mjcf.compiler's (masses, inertias, body / geom frames, joint ranges, gears);
  2. puts MuJoCo, the oracle (and the device engine) into the same seeded state and applies the same torque script
     (gravity compensation + a seeded sinusoid on the arm, a square wave on the gripper actuators) for --steps substeps of mj_step;
  3. reports, per step, |qpos|, |qvel| differences, ncon, nefc and the contact-force sum, and fails (exit 1) when the divergence over the first
     --gate-steps substeps exceeds --tol (default 1e-6 for 50 substeps: contact-rich trajectories are chaotic, so only the early window is
     gated; the full curve is printed for inspection).
Prints one JSON object; exit code 0 = within tolerance, 1 = mismatch, 2 = mujoco not importable."""
import argparse
import json
import os
import re
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

REF_ASSET_PREFIX = "/root/reference/robosuite/models/assets"
TASKS = ["Lift_Panda", "Lift_Sawyer", "Stack_Panda", "Door_Panda", "PickPlace_Panda", "NutAssemblyRound_Panda"]


def load_mjcf(task, assets):
    """fixture MJCF with the recorded asset prefix replaced and every texture / textured material attribute removed"""
    xml = open(os.path.join(ROOT, "tests", "golden", "mjcf", task + ".xml")).read()
    xml = re.sub(r"<texture\b[^>]*/>", "", xml)
    xml = re.sub(r'\stexture="[^"]*"', "", xml)
    xml = re.sub(r'\s(texrepeat|texuniform)="[^"]*"', "", xml)
    return xml.replace(REF_ASSET_PREFIX, os.path.abspath(assets))


def seeded_state(model, seed):
    """a reset-like state: qpos0 with N(0, 0.02^2) on the arm joints (robots/robot.py:247-259)"""
    rng = np.random.default_rng(seed)
    q = np.array(model.qpos0, dtype=np.float64)
    arm = [i for i, n in enumerate(model.names["joint"]) if n and n.startswith("robot0_")]
    for j in arm:
        q[int(model.jnt_qposadr[j])] += rng.normal(0, 0.02)
    return q


def torque_script(nu, n_arm, steps, seed):
    """[steps, nu] offsets added to gravity compensation: sinusoids on the arm, +-1 square wave (actuator ctrl units) on the gripper"""
    rng = np.random.default_rng(seed + 1)
    t = np.arange(steps)[:, None] * 0.002
    amp, freq, ph = rng.uniform(0.5, 4.0, n_arm), rng.uniform(0.2, 1.5, n_arm), rng.uniform(0, 2 * np.pi, n_arm)
    out = np.zeros((steps, nu))
    out[:, :n_arm] = amp * np.sin(2 * np.pi * freq * t + ph)
    if nu > n_arm:
        sq = np.where((np.arange(steps) // 150) % 2 == 0, -1.0, 1.0)[:, None]
        sign = np.array([1.0 if k % 2 == 0 else -1.0 for k in range(nu - n_arm)])
        out[:, n_arm:] = sq * sign
    return out


def compare_constants(mm, model):
    out = {}

    def d(name, a, b):
        if a is None:
            return
        a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
        out[name] = float(np.abs(a.reshape(-1) - b.reshape(-1)).max()) if a.size == b.size else f"shape {a.shape} vs {b.shape}"
    for k in ("nq", "nv", "nu", "nbody", "ngeom", "njnt"):
        out[k] = [int(getattr(mm, k)), int(getattr(model, k))]
    d("body_mass", mm.body_mass, model.body_mass)
    d("body_inertia", mm.body_inertia, model.body_inertia)
    d("body_pos", mm.body_pos, model.body_pos)
    d("body_quat", mm.body_quat, model.body_quat)
    d("body_ipos", mm.body_ipos, model.body_ipos)
    d("body_iquat_abs", np.abs(mm.body_iquat), np.abs(model.body_iquat))
    d("jnt_range", mm.jnt_range, model.jnt_range)
    d("dof_damping", mm.dof_damping, model.dof_damping)
    d("dof_armature", mm.dof_armature, model.dof_armature)
    d("dof_frictionloss", mm.dof_frictionloss, model.dof_frictionloss)
    d("geom_size", mm.geom_size, model.geom_size)
    d("geom_pos", mm.geom_pos, model.geom_pos)
    d("geom_friction", mm.geom_friction, model.geom_friction)
    d("actuator_gear", mm.actuator_gear[:, 0], np.asarray(model.actuator_gear).reshape(model.nu, -1)[:, 0])
    d("qpos0", mm.qpos0, model.qpos0)
    return out


def run_task(task, args):
    import mujoco

    from oracle.pyoracle import Oracle
    from robosuite_b200.mjcf.compiler import load_model, pack_model

    model = load_model(os.path.join(ROOT, "tests", "golden", "models", task + ".npz"))
    mm = mujoco.MjModel.from_xml_string(load_mjcf(task, args.assets))
    md = mujoco.MjData(mm)
    res = {"task": task, "constants_max_abs_diff": compare_constants(mm, model)}
    q0 = seeded_state(model, args.seed)
    n_arm = len([n for n in model.names["actuator"] if n and n.startswith("robot0_")])
    script = torque_script(model.nu, n_arm, args.steps, args.seed)

    o = Oracle(pack_model(model))
    o.reset_data()
    o.qpos[:] = q0
    o.qvel[:] = 0
    o.forward()
    md.qpos[:] = q0
    md.qvel[:] = 0
    mujoco.mj_forward(mm, md)
    dev = None
    if args.device:
        import torch

        from robosuite_b200.engine import BatchedSim

        dev = BatchedSim(model, 1, device=0, precision="f64")
        dev.qpos[:] = torch.as_tensor(q0, device=dev.torch_device)
        dev.qvel[:] = 0
        dev.forward()
    arm_dofs = [int(model.jnt_dofadr[j]) for j, n in enumerate(model.names["joint"]) if n and n.startswith("robot0_")][:n_arm]
    curve = []
    for t in range(args.steps):
        # the same control on every engine, computed from MuJoCo's own bias so that a divergence of the states does not feed back into the input
        u = script[t].copy()
        u[:n_arm] += md.qfrc_bias[arm_dofs]
        lo, hi = np.asarray(model.actuator_ctrlrange)[:, 0], np.asarray(model.actuator_ctrlrange)[:, 1]
        lim = np.asarray(model.actuator_ctrllimited).astype(bool)
        u = np.where(lim, np.clip(u, lo, hi), u)
        md.ctrl[:] = u
        o.ctrl[:] = u
        mujoco.mj_step(mm, md)
        o.step()
        row = {"t": t, "ncon": [int(md.ncon), int(o.ncon)], "nefc": [int(getattr(md, "nefc", -1)), int(o.nefc)],
               "dq_oracle": float(np.abs(md.qpos - o.qpos).max()), "dv_oracle": float(np.abs(md.qvel - o.qvel).max()),
               "dfc_oracle": float(np.abs(md.qfrc_constraint - o.qfrc_constraint).max())}
        if dev is not None:
            import torch

            dev.ctrl[:] = torch.as_tensor(u, device=dev.torch_device)
            dev.step(1)
            row["dq_device"] = float(np.abs(md.qpos - dev.qpos[0].cpu().numpy()).max())
            row["dv_device"] = float(np.abs(md.qvel - dev.qvel[0].cpu().numpy()).max())
        curve.append(row)
    g = curve[:args.gate_steps]
    res["gate"] = {"steps": args.gate_steps, "tol": args.tol,
                   "max_dq_oracle": max(r["dq_oracle"] for r in g), "max_dv_oracle": max(r["dv_oracle"] for r in g),
                   "ncon_equal": all(r["ncon"][0] == r["ncon"][1] for r in g)}
    if dev is not None:
        res["gate"]["max_dq_device"] = max(r["dq_device"] for r in g)
    res["ok"] = bool(res["gate"]["max_dq_oracle"] <= args.tol and res["gate"]["ncon_equal"]
                     and (dev is None or res["gate"]["max_dq_device"] <= args.tol))
    res["curve_every_25"] = curve[::25]
    res["final"] = curve[-1]
    return res


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--assets", default=None, help="robosuite/models/assets of an installed robosuite (meshes of the robots and objects)")
    ap.add_argument("--tasks", nargs="*", default=TASKS)
    ap.add_argument("--steps", type=int, default=250)
    ap.add_argument("--gate-steps", type=int, default=50)
    ap.add_argument("--tol", type=float, default=1e-6)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--device", action="store_true", help="also run the CUDA engine (f64, 1 env)")
    args = ap.parse_args(argv)
    try:
        import mujoco  # noqa: F401
    except ImportError:
        print(json.dumps({"unavailable": "mujoco is not importable here (pip install mujoco on a networked machine)"}))
        return 2
    if args.assets is None:
        try:
            import robosuite

            args.assets = os.path.join(os.path.dirname(robosuite.__file__), "models", "assets")
        except ImportError:
            ap.error("--assets is required when robosuite is not installed")
    results = [run_task(t, args) for t in args.tasks]
    print(json.dumps({"mujoco": __import__("mujoco").__version__, "results": results}, indent=1))
    return 0 if all(r["ok"] for r in results) else 1


if __name__ == "__main__":
    sys.exit(main())
