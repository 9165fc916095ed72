"""Device time of one Lift/Panda control step (env.step) with and without one of the array-group exports, f32, CUDA events around K
steps after W warm-up steps, random actions.  KIND is the group: contacts (the contact records), step1 (the step-1 arrays) or
step2 (the step-2 arrays).  Configurations, alternated over R rounds so that their spread can be read beside their difference:
  pipeline            the pipeline schedule, no export (the default);
  pipeline+<group>    the pipeline with the group's export: make(contact_queries=True), make(data_queries=True), or
                      make(dynamics_queries=True) (the step-2 export and the contact records);
  pipeline+query      the same plus one query per step, its torch ops (and for step1 the Jacobian kernel) on the step's stream:
                      contacts env._check_grasp(cube); step1 sim.data.get_site_xpos and get_site_jacp of the end-effector site;
                      step2 sim.data.contact_force() and an actuator_force read;
  unit+contacts       (contacts only) the unit queue (mode 2) with the contact export;
  fused+full_export   set_export(True): what delivered the group before its export - the fused kernel writing every derived array
                      (poses, qM, cdof, contacts, efc rows, actuator forces) on the last substep.
Prints one JSON line per configuration and round, with the card's name and power limit (contacts: also the mean ncon).
usage: python tools/probe_exports.py {contacts|step1|step2} [n_env=4096] [steps=20] [warmup=5] [rounds=3]"""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import robosuite_b200 as suite  # noqa: E402

KIND = sys.argv[1] if len(sys.argv) > 1 else ""
n = int(sys.argv[2]) if len(sys.argv) > 2 else 4096
K = int(sys.argv[3]) if len(sys.argv) > 3 else 20
W = int(sys.argv[4]) if len(sys.argv) > 4 else 5
R = int(sys.argv[5]) if len(sys.argv) > 5 else 3


def query_contacts(env):
    grasped = torch.zeros(n, dtype=torch.long, device=env.device)
    return lambda: grasped.add_(env._check_grasp(env.cube_geoms).long())


def query_step1(env):
    acc = torch.zeros((n, 3), dtype=env.dtype, device=env.device)
    site = env.eef_site_id

    def q():
        acc.add_(env.sim.data.get_site_xpos(site))
        acc.add_(env.sim.data.get_site_jacp(site)[:, :, 0])
    return q


def query_step2(env):
    acc = torch.zeros((n, 6), dtype=env.dtype, device=env.device)

    def q():
        acc.add_(env.sim.data.contact_force().sum(1))
        acc[:, 0].add_(env.sim.data.actuator_force[:, 0])
    return q


# per kind: the make() switch of its export, the query, and whether the unit queue is measured too
KINDS = {"contacts": ("contact_queries", query_contacts, True), "step1": ("data_queries", query_step1, False),
         "step2": ("dynamics_queries", query_step2, False)}
if KIND not in KINDS:
    sys.exit(__doc__.splitlines()[-1])
switch, make_query, unit = KINDS[KIND]
on = {switch: True}
CONFIGS = {"pipeline": dict(kw={}), "pipeline+" + KIND: dict(kw=on), "pipeline+query": dict(kw=on, query=True)}
if unit:
    CONFIGS["unit+" + KIND] = dict(kw=on, mode=2)
CONFIGS["fused+full_export"] = dict(kw={}, full=True)
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                   capture_output=True, text=True).stdout.strip().split(", ")


def measure(cfg):
    env = suite.make("Lift", robots="Panda", num_envs=n, seed=1, horizon=10 ** 9, precision="f32", **cfg["kw"])
    if "mode" in cfg:
        env.sim.set_mode(cfg["mode"])
    if cfg.get("full"):
        env.sim.set_export(True)
    gen = torch.Generator(device=env.device)
    gen.manual_seed(3)
    acts = torch.rand((W + K, n, env.action_dim), generator=gen, device=env.device, dtype=env.dtype) * 2 - 1
    query = make_query(env) if cfg.get("query") else None

    def step(a):
        env.step(a)
        if query:
            query()

    for k in range(W):
        step(acts[k])
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for k in range(W, W + K):
        step(acts[k])
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / K
    ncon = float(env.sim.ncon.float().mean()) if KIND == "contacts" and (cfg["kw"] or cfg.get("full")) else None
    env.close()
    return ms, ncon


for r in range(R):
    for name, cfg in CONFIGS.items():
        ms, ncon = measure(cfg)
        line = {"config": name, "round": r, "n_env": n, "steps": K, "ms_per_step": round(ms, 3),
                "env_steps_per_s": round(n * 1000.0 / ms)}
        if KIND == "contacts":
            line["mean_ncon_last_substep"] = ncon
        line.update(gpu=q[0], power_limit=q[1] if len(q) > 1 else None)
        print(json.dumps(line), flush=True)
