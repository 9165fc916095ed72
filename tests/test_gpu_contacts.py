"""GPU: the contact export (b2s_set_contact_export, BatchedSim.contacts) and the environment's contact queries (every schedule
writing the full export's records: tests/test_gpu_exports.py).

* in f64 the records match the CPU oracle's data.contact (pairs and order exactly, geometry to 1e-12);
* check_contact / get_contacts / _check_grasp equal the numpy restatement of the reference (tests/contact_ref.py) on the exported
  arrays, and _check_grasp of the task object equals the device's own grasp flag on the recorded grasp episodes;
* the errors."""
import numpy as np
import pytest

from tests import contact_ref as ref
from tests.oracle_sim_export import ExportOracleSim
from tests.schedules import make_env, random_actions

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

TASKS = ["Lift", "Stack", "Door", "NutAssemblyRound", "PickPlace"]


def _sync(cpu, dev):
    """the CPU stand-in takes the device's state: everything the next substep reads"""
    def f64(x):
        return x.detach().cpu().to(torch.float64)

    cs, ds = cpu.sim, dev.sim
    cs.qpos[:] = f64(ds.qpos); cs.qvel[:] = f64(ds.qvel); cs.qacc_warmstart[:] = f64(ds.qacc_warmstart)
    cs.ctrl[:] = f64(ds.ctrl); cs.time[:] = f64(ds.time)
    gp, go, ij, gs = f64(ds.ctrl_goal_pos), f64(ds.ctrl_goal_ori), f64(ds.ctrl_initial_joint), f64(ds.ctrl_grip_state)
    for e in range(dev.num_envs):
        st = cs.o[e].ctrl_state
        for k in range(3):
            st.goal_pos[k] = float(gp[e, k])
        for k in range(9):
            st.goal_ori[k] = float(go[e, k])
        for k in range(8):
            st.initial_joint[k] = float(ij[e, k])
        for k in range(4):
            st.grip_action[k] = float(gs[e, k])
    if getattr(dev, "_door_ov", None) is not None:  # the Door's per-environment placement
        for (dp, dq), (cp, cq) in zip(dev._door_ov, cpu._door_ov):
            cp[:] = f64(dp); cq[:] = f64(dq)


@pytest.mark.parametrize("task", TASKS)
def test_records_match_the_oracle_in_f64(task):
    """before every comparison the CPU stand-in takes the device's state; both then run one substep (env_step with n_substeps = 1,
    whose contacts are those of its step1).  Between comparisons the device runs whole control steps on its own."""
    import robosuite_b200 as suite

    n = 4
    kw = dict(robots="Panda", num_envs=n, seed=11, contact_queries=True)
    dev = suite.make(task, precision="f64", **kw)
    cpu = suite.make(task, sim_cls=ExportOracleSim, precision="f64", **kw)
    rng = np.random.default_rng(2)
    knife = compared = 0
    for t in range(5):
        act = rng.uniform(-1, 1, size=(n, dev.action_dim))
        act[:, :3] = [0, 0, -1] if t >= 2 else act[:, :3]
        _sync(cpu, dev)
        dev.sim.env_step(torch.as_tensor(act, device=dev.device).contiguous(), 1)
        cpu.sim.env_step(torch.as_tensor(act), 1)
        torch.cuda.synchronize()
        d = {k: v.cpu() for k, v in dev.sim.contacts().items()}
        c = cpu.sim.contacts()
        for e in range(n):
            nd, nc = int(d["ncon"][e]), int(c["ncon"][e])
            pd, pc = d["geom"][e, :nd].tolist(), c["geom"][e, :nc].tolist()
            if pd != pc:  # DESIGN section 3: a pair at exactly zero depth may be active in one engine only
                knife += 1
                only_d = [float(d["dist"][e, k]) for k in range(nd) if pd[k] not in pc]
                only_c = [float(c["dist"][e, k]) for k in range(nc) if pc[k] not in pd]
                assert only_d + only_c and all(abs(x) < 1e-9 for x in only_d + only_c), (task, t, e, pd, pc)
                continue
            assert (d["geom"][e, nd:] == -1).all()
            compared += 1
            # a mesh resting face-down on a face has a plane of deepest points: the convex narrow phase returns one of them, and
            # which one depends on the order of the support scan (the same depth and normal, another point): pos is compared for
            # the other pairs only
            mesh = [k for k in range(nd) if 7 in (int(dev.model.geom_type[pd[k][0]]), int(dev.model.geom_type[pd[k][1]]))]
            for f in ("dist", "pos", "frame", "friction"):
                rows = [k for k in range(nd) if f != "pos" or k not in mesh]
                err = float((d[f][e, rows] - c[f][e, rows]).abs().max()) if rows else 0.0
                assert err < 1e-12, (task, t, e, f, err)
        dev.step(torch.as_tensor(act, device=dev.device))
    assert compared >= 4 * n and knife <= n, (compared, knife)
    dev.close()
    cpu.close()


@pytest.mark.parametrize("task", TASKS)
def test_queries_equal_the_restatement(task):
    env = make_env(task, 8, 1, 4, contact_queries=True)
    m = env.model
    gn = m.names["geom"]
    colliding = sorted({int(g) for p in m.pair_geom for g in p})
    robot, grip = env.contact_geoms("robot0_"), env.contact_geoms("gripper0_")
    objects = [g for g in colliding if not (gn[g] or "").startswith(("robot0_", "gripper0_", "fixed_mount0_"))]
    left, right = env._fingerpad_geoms()
    sets = [(robot, None), (grip, None), (grip, objects), (objects, robot), (left, objects), (objects, None)]
    acts = random_actions(env, 5, seed=1)
    seen = 0
    for t in range(5):
        a = acts[t].clone()
        if t >= 2:
            a[:, 2] = -1  # down onto the objects
        env.step(a)
        c = {k: v.cpu() for k, v in env.sim.contacts().items()}
        seen += int(c["ncon"].sum())
        for x, y in sets:
            got = env.check_contact(x, y).cpu().tolist()
            assert got == [ref.check_contact(m, c["ncon"][e], c["geom"][e], x, y) for e in range(8)], (task, t, x, y)
            g = env.get_contacts(x).cpu().numpy()
            for e in range(8):
                assert np.array_equal(g[e], ref.get_contacts(m, c["ncon"][e], c["geom"][e], x)), (task, t, e, x)
        got = env._check_grasp(objects).cpu().tolist()
        assert got == [ref.check_grasp(m, c["ncon"][e], c["geom"][e], [left, right], objects) for e in range(8)]
        # device tensors of ids are used as they are
        ids = torch.as_tensor(grip, device=env.device)
        assert torch.equal(env.check_contact(ids, objects), env.check_contact(grip, objects))
    assert task == "Door" or seen > 0  # the door is touched only by chance
    env.close()


@pytest.mark.parametrize("key", ["Lift", "Stack"])
def test_check_grasp_is_the_task_grasp_flag_on_the_grasp_episodes(key):
    import robosuite_b200 as suite
    from tests.test_gpu_task_logic import _case

    task, kw, m, rec = _case(key)
    env = suite.make(task, robots="Panda", num_envs=1, seed=0, horizon=1000, model=m, contact_queries=True, **kw)
    env.reset_to(rec["qpos0"])
    obj = env.cube_geoms if task == "Lift" else env.cubeA_geoms
    grasped = 0
    for a in rec["actions"]:
        env.step(torch.as_tensor(a[None]))
        flag = env._check_grasp(obj)
        assert bool(flag[0]) == bool(env.sim.task_out[0, 2] > 0)
        grasped += int(flag[0])
    assert grasped > 0
    env.close()


def test_errors():
    from robosuite_b200.engine import lib

    env = make_env("Lift", 2, 1, 0)
    env.step(torch.zeros((2, env.action_dim), device=env.device))
    for call in (lambda: env.check_contact("cube_g0"), lambda: env.get_contacts("cube_g0"), lambda: env._check_grasp("cube_g0")):
        with pytest.raises(RuntimeError, match="contact_queries"):
            call()
    L = lib()
    assert L.b2s_set_contact_export(None, 1) == -1
    assert b"null handle" in L.b2s_last_error()
    assert L.b2s_set_contact_export(env.sim._h, 1) == 0 and L.b2s_set_contact_export(env.sim._h, 0) == 0
    env.close()
