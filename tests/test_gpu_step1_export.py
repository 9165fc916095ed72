"""GPU: the step-1 export (b2s_set_step1_export, BatchedSim.set_step1_export, make(..., data_queries=True)) and the batched
MjData view.

* the pipeline (with the default group count and with one group) and the unit queue write the same step-1 arrays as the fused
  kernel with the full export, bit for bit, through a masked reset and with a small tier that sends environments to the large one;
* the Jacobians (b2s_jac_site / jac_body / jac_geom) and b2s_full_m read from them equal those after the full export;
* switching the export on changes no other output in any schedule;
* sim.data reads the poses the observations read;
* the errors."""
import pytest

from tests.schedules import make_env, random_actions, switches

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

TASKS = ["Lift", "Stack", "Door", "NutAssemblyRound", "PickPlace"]
STATE = ("qpos", "qvel", "qacc", "ctrl", "obs", "task_out", "warn")
STEP1 = ("xpos", "xquat", "xmat", "site_xpos", "site_xmat", "geom_xpos", "geom_xmat", "qM", "cdof", "qfrc_bias", "qfrc_passive")
TIER = (4, 20)  # small-tier capacities (contacts, rows): a cube resting on the table already needs more rows (4 contacts, 21 rows)


def _rollout(task, precision, mode, export, groups=None, n=16, steps=6):
    """outputs after every step (and the masked reset before step 3).  export: None, "step1" (make(data_queries=True)) or "full"
    (set_export(True): the fused kernel with every derived array).  Returns (states, arrays): states = the contact records (ncon
    first; the contact export is on in every run), the STATE fields and task_vec; arrays = the step-1 arrays, then the Jacobians of the
    end-effector site, the last body and the first colliding geom and full_m, then nefc with the full export"""
    with switches(gjk_cache=False, ctrl_split=False, groups=groups):
        env = make_env(task, n, mode, 5, groups=groups, gjk_cache=False, ctrl_split=False, tier_small=TIER, precision=precision,
                       contact_queries=True, data_queries=export == "step1")
        sim = env.sim
        if export == "full":
            sim.set_export(True)
        geom = min(int(g) for p in env.model.pair_geom for g in p)
        acts = random_actions(env, steps)
        acts[2:, : n // 2, 2] = -1  # half of the arms push down onto the table and the objects: more contacts
        fields = STATE + (("task_vec",) if hasattr(sim, "task_vec") else ())
        states, arrays = [], []

        def record():
            states.append([t.clone() for t in sim.contacts().values()] + [getattr(sim, f).clone() for f in fields])
            if export:
                jac = [*sim.jac_site(env.eef_site_id), *sim.jac_body(env.model.nbody - 1), *sim.jac_geom(geom), sim.full_m()]
                arrays.append([getattr(sim, f).clone() for f in STEP1] + jac + ([sim.nefc.clone()] if export == "full" else []))

        for t in range(steps):
            if t == steps // 2:
                mask = torch.zeros(n, dtype=torch.bool, device=env.device)
                mask[::3] = True
                env.reset(mask=mask)
                record()
            env.step(acts[t])
            record()
        torch.cuda.synchronize()
        env.close()
    return states, arrays


def _equal(a, b, tag):
    assert len(a) == len(b), tag
    for k, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x, y), (tag, k)


@pytest.mark.parametrize("precision", ["f32", "f64"])
@pytest.mark.parametrize("task", TASKS)
def test_schedules_write_the_fused_kernels_arrays(task, precision):
    s_full, full = _rollout(task, precision, 0, "full")
    # environments whose last substep did not fit the small tier ran in the large one; the Door's arms touch the door only by
    # chance, and its environments stay in the small tier
    over = torch.stack([(s[0] > TIER[0]) | (a[-1] > TIER[1]) for s, a in zip(s_full, full)])
    assert task == "Door" or bool(over.any()), task
    # the arrays are fresh after every step: the poses move
    assert all(not torch.equal(full[t][0], full[t + 1][0]) for t in range(len(full) - 1))
    full = [a[:-1] for a in full]
    for mode, groups in ((0, None), (1, None), (1, 1), (2, None)):
        s_off, _ = _rollout(task, precision, mode, None, groups)
        s_on, arr = _rollout(task, precision, mode, "step1", groups)
        for t, (a, b) in enumerate(zip(s_off, s_on)):
            _equal(a, b, (task, precision, mode, groups, "state", t))
        for t, (a, b) in enumerate(zip(full, arr)):
            _equal(a, b, (task, precision, mode, groups, "step1", t))


def test_data_reads_the_poses_the_observations_read():
    env = make_env("Lift", 64, 1, 2, data_queries=True)
    d = env.sim.data
    acts = random_actions(env, 3, seed=4)
    for a in acts:
        obs, _, _, _ = env.step(a)
        assert torch.equal(obs["robot0_eef_pos"], d.get_site_xpos("gripper0_right_grip_site"))
        assert torch.equal(obs["cube_pos"], d.get_body_xpos("cube_main"))
        v = d.get_site_xvelp(env.eef_site_id)
        assert torch.equal(v, (d.get_site_jacp(env.eef_site_id) @ env.sim.qvel[:, :, None])[:, :, 0])
        assert torch.equal(d.full_m(), d.qM)
    env.close()


def test_errors():
    from robosuite_b200.engine import lib

    env = make_env("Lift", 2, 1, 0)
    env.step(torch.zeros((2, env.action_dim), device=env.device))
    for call in (lambda: env.sim.data.body_xpos, lambda: env.sim.data.get_site_jacp(0), lambda: env.sim.data.full_m()):
        with pytest.raises(RuntimeError, match="data_queries"):
            call()
    L = lib()
    assert L.b2s_set_step1_export(None, 1) == -1
    assert b"null handle" in L.b2s_last_error()
    assert L.b2s_set_step1_export(env.sim._h, 1) == 0 and L.b2s_set_step1_export(env.sim._h, 0) == 0
    env.close()
