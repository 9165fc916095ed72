"""GPU: every schedule writes the array groups the last substep of a step call exports (the contact records, b2s_set_contact_export;
the step-1 arrays, b2s_set_step1_export; the step-2 arrays, b2s_set_step2_export) with the full export's bits, and switching a
group on changes nothing else.

* The fused kernel, the pipeline (with the default group count and with one group) and the unit queue each run the chain of
  exports (), (contacts), (contacts, step1), (contacts, step1, step2) through a masked reset and with a small tier that sends
  environments to the large one.  Each link leaves every output of the one before it bit-identical (state, observations, task
  rows, and the groups both have on), and each group's arrays equal those of the fused kernel with the full export, bit for bit:
  the step-1 arrays together with the Jacobians (b2s_jac_site / jac_body / jac_geom) and b2s_full_m read from them, the step-2
  arrays with the valid constraint rows only.
* In the default configuration (GJK warm start on, OSC a phase-1 role, no small-tier override) the step-2 export changes no other
  output in any schedule."""
import pytest

from tests.schedules import make_env, random_actions, switches

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

TASKS = ["Lift", "Stack", "Door", "NutAssemblyRound", "PickPlace"]
STATE = ("qpos", "qvel", "qacc", "ctrl", "obs", "task_out", "warn")
STEP1 = ("xpos", "xquat", "xmat", "site_xpos", "site_xmat", "geom_xpos", "geom_xmat", "qM", "cdof", "qfrc_bias", "qfrc_passive")
STEP2 = ("qfrc_actuator", "actuator_force", "qfrc_smooth", "qacc_smooth", "qfrc_constraint", "nefc", "solver_niter",
         "contact_efc_address")
ROWS = ("efc_type", "efc_D", "efc_R", "efc_aref", "efc_force")
GROUPS = ("contacts", "step1", "step2")
TIER = (4, 20)  # small-tier capacities (contacts, rows): a cube resting on the table already needs more rows (4 contacts, 21 rows)


def _contacts(env):
    return [t.clone() for t in env.sim.contacts().values()]  # ncon first


def _step1(env):
    """the step-1 arrays, then the Jacobians of the end-effector site, the last body and the first colliding geom, and full_m"""
    sim = env.sim
    geom = min(int(g) for p in env.model.pair_geom for g in p)
    jac = [*sim.jac_site(env.eef_site_id), *sim.jac_body(env.model.nbody - 1), *sim.jac_geom(geom), sim.full_m()]
    return [getattr(sim, f).clone() for f in STEP1] + jac


def _step2(env):
    """the step-2 arrays with only the valid rows of efc_* (the first nefc, and the first nefc * nv of efc_J), flattened"""
    sim = env.sim
    nefc = sim.nefc.long()
    out = [getattr(sim, f).clone() for f in STEP2]
    me = sim.efc_force.shape[1]
    rows = torch.arange(me, device=nefc.device)[None, :] < nefc[:, None]
    out += [getattr(sim, f)[rows].clone() for f in ROWS]
    J = sim.efc_J.reshape(sim.efc_J.shape[0], -1)
    out.append(J[torch.arange(J.shape[1], device=nefc.device)[None, :] < (nefc * sim.model.nv)[:, None]].clone())
    return out


READ = {"contacts": _contacts, "step1": _step1, "step2": _step2}


def _rollout(task, precision, mode, groups, exports, default=False, n=16, steps=6):
    """outputs after every step (and the masked reset before step 3).  exports: "full" (set_export(True): the fused kernel with every
    derived array; the queries on too) or a tuple of GROUPS (make(contact_queries / data_queries / dynamics_queries=True)).
    default: the library's default configuration (GJK warm start, OSC role, no small-tier override).  Returns (states, arrays):
    states = the STATE fields and task_vec; arrays = {group: its READ list} for each group that is on"""
    on = GROUPS if exports == "full" else exports
    sw = dict(gjk_cache=default, ctrl_split=default, groups=groups)
    with switches(**sw):
        env = make_env(task, n, mode, 5, tier_small=None if default else TIER, precision=precision,
                       contact_queries="contacts" in on, data_queries="step1" in on, dynamics_queries="step2" in on, **sw)
        sim = env.sim
        if exports == "full":
            sim.set_export(True)
        acts = random_actions(env, steps)
        acts[2:, : n // 2, 2] = -1  # half of the arms push down onto the table and the objects: more contacts
        fields = STATE + (("task_vec",) if hasattr(sim, "task_vec") else ())
        states, arrays = [], []

        def record():
            states.append([getattr(sim, f).clone() for f in fields])
            arrays.append({g: READ[g](env) for g in on})

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


def _same(ref, run, groups, tag):
    """the states of two rollouts, and the arrays of `groups`, bit-identical after every step"""
    for t, (a, b) in enumerate(zip(ref[0], run[0])):
        _equal(a, b, tag + ("state", t))
    for g in groups:
        for t, (a, b) in enumerate(zip(ref[1], run[1])):
            _equal(a[g], b[g], tag + (g, t))


@pytest.mark.parametrize("precision", ["f32", "f64"])
@pytest.mark.parametrize("task", TASKS)
def test_schedules_write_the_fused_kernels_arrays(task, precision):
    _, full = _rollout(task, precision, 0, None, "full")
    # environments whose last substep did not fit the small tier (more contacts or rows than it holds) ran in the large one; the
    # Door's arms touch the door only by chance, and its environments stay in the small tier
    nefc_at = STEP2.index("nefc")
    over = torch.stack([(a["contacts"][0] > TIER[0]) | (a["step2"][nefc_at] > TIER[1]) for a in full])
    assert task == "Door" or bool(over.any()), task
    # the arrays are fresh after every step: the poses move and the forces change
    for g in ("step1", "step2"):
        assert all(not torch.equal(full[t][g][0], full[t + 1][g][0]) for t in range(len(full) - 1)), g
    for mode, groups in ((0, None), (1, None), (1, 1), (2, None)):
        prev = None
        for k in range(len(GROUPS) + 1):
            exports = GROUPS[:k]
            run = _rollout(task, precision, mode, groups, exports)
            tag = (task, precision, mode, groups, exports)
            if prev is not None:
                _same(prev, run, GROUPS[:k - 1], tag)
            for g in exports:
                for t, (a, b) in enumerate(zip(full, run[1])):
                    _equal(a[g], b[g], tag + ("full", g, t))
            prev = run


@pytest.mark.parametrize("precision", ["f32", "f64"])
@pytest.mark.parametrize("task", TASKS)
def test_flag_changes_nothing_else_in_the_default_configuration(task, precision):
    for mode in (0, 1, 2):
        off = _rollout(task, precision, mode, None, ("contacts", "step1"), default=True)
        on = _rollout(task, precision, mode, None, GROUPS, default=True)
        _same(off, on, ("contacts", "step1"), (task, precision, mode, "default"))
