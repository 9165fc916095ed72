"""Single-object PickPlace / NutAssembly variants (single_object_mode 1 and 2) on the CPU stand-in (tests/oracle_sim_select.py):
names, observation layouts, reset states, the mode-1 draw, the selected-object rows, and the reward / success rules restated in
numpy."""
import math

import numpy as np
import pytest
import torch

import robosuite_b200 as suite
from robosuite_b200.envs.base import SIM_WARN_BITS
from tests.oracle_sim_select import SelectOracleSim

PROPRIO = 50
REL = ("_to_robot0_eef_pos", 3), ("_to_robot0_eef_quat", 4), ("_pos", 3), ("_quat", 4)
# the `object` modality of every new name, in observation order: (key, width)
OBJECT_KEYS = {
    "PickPlaceMilk": [("Milk" + s, w) for s, w in REL],
    "PickPlaceBread": [("Bread" + s, w) for s, w in REL],
    "PickPlaceCereal": [("Cereal" + s, w) for s, w in REL],
    "PickPlaceCan": [("Can" + s, w) for s, w in REL],
    "PickPlaceSingle": [("obj" + s, w) for s, w in REL] + [("obj_id", 1)],
    "NutAssemblySingle": [("nut" + s, w) for s, w in REL] + [("nut_id", 1)],
}


def _make(task, n=2, seed=0, **kw):
    return suite.make(task, robots="Panda", num_envs=n, seed=seed, sim_cls=SelectOracleSim, precision="f64", **kw)


def _actions(env, k, seed=0):
    rng = np.random.default_rng(seed)
    return [torch.as_tensor(rng.uniform(-1, 1, size=(env.num_envs, env.action_dim))) for _ in range(k)]


@pytest.mark.parametrize("task", sorted(OBJECT_KEYS))
def test_new_names_build_with_the_reference_observation_layout(task):
    env = _make(task)
    keys = list(env._obs_slices)
    obj = [k for k in keys if k not in keys[:10]]
    assert [(k, env._obs_slices[k][1] - env._obs_slices[k][0]) for k in obj] == OBJECT_KEYS[task]
    width = sum(w for _, w in OBJECT_KEYS[task])
    assert env.obs_dim == PROPRIO + width
    assert env._modality_slices["object-state"] == (PROPRIO, PROPRIO + width)
    obs = env._get_observations()
    assert obs["object-state"].shape == (2, width)


def _rollout(env, k=3, seed=0):
    out = []
    for a in _actions(env, k, seed):
        obs, r, d, _ = env.step(a)
        out.append((env.sim.obs.clone(), r.clone(), env.sim.qpos.clone()))
    return out


@pytest.mark.parametrize("kw, name", [(dict(task="PickPlace", single_object_mode=2, object_type="can"), "PickPlaceCan"),
                                      (dict(task="NutAssembly", single_object_mode=2, nut_type="round"), "NutAssemblyRound")])
def test_mode2_keywords_equal_the_registered_class(kw, name):
    kw = dict(kw)
    a = _make(kw.pop("task"), seed=5, reward_shaping=True, **kw)
    b = _make(name, seed=5, reward_shaping=True)
    assert list(a._obs_slices) == list(b._obs_slices)
    assert torch.equal(a.sim.obs, b.sim.obs) and torch.equal(a.sim.qpos, b.sim.qpos)
    for (oa, ra, qa), (ob, rb, qb) in zip(_rollout(a), _rollout(b)):
        assert torch.equal(oa, ob) and torch.equal(ra, rb) and torch.equal(qa, qb)


def _obj_qpos(env, q, name):
    a = env.obj_qadr[name]
    return q[:, a:a + 7]


def test_reset_states_parked_objects_and_mode2_placement():
    base = _make("PickPlace", n=3, seed=9)
    q0 = base.sim.qpos
    for i, t in enumerate(("Milk", "Bread", "Cereal", "Can")):
        env = _make("PickPlace" + t, n=3, seed=9)
        q = env.sim.qpos
        for j, other in enumerate(env.obj_names):
            if j == i:  # same draws as mode 0: the active object's placement is mode 0's
                assert torch.equal(_obj_qpos(env, q, other), _obj_qpos(base, q0, other))
            else:
                assert torch.equal(_obj_qpos(env, q, other), torch.tensor([[10.0, 10, 10, 1, 0, 0, 0]] * 3, dtype=q.dtype))
        assert env.object_id == i
    single = _make("PickPlaceSingle", n=3, seed=9)
    q, sel = single.sim.qpos, single.object_id
    for e in range(3):
        for j, other in enumerate(single.obj_names):
            if j == int(sel[e]):
                assert torch.equal(_obj_qpos(single, q, other)[e], _obj_qpos(base, q0, other)[e])
            else:
                assert torch.equal(_obj_qpos(single, q, other)[e], torch.tensor([10.0, 10, 10, 1, 0, 0, 0], dtype=q.dtype))
    nut = _make("NutAssemblySingle", n=3, seed=9)
    for e in range(3):
        k = int(nut.object_id[e])
        parked = _obj_qpos(nut, nut.sim.qpos, nut.nut_names[1 - k])[e]
        assert torch.equal(parked, torch.tensor([10.0, 10, 10, 1, 0, 0, 0], dtype=parked.dtype))


@pytest.mark.parametrize("task, k", [("PickPlaceSingle", 4), ("NutAssemblySingle", 2)])
def test_mode1_draw_is_uniform(task, k):
    from scipy.stats import chisquare

    env = _make(task, n=2, seed=1)
    env._sample_reset_state(4096)
    counts = np.bincount(env._sel_draw.numpy(), minlength=k)
    assert len(counts) == k
    assert chisquare(counts).pvalue > 1e-3, counts


def test_masked_reset_redraws_only_the_masked_environments():
    env = _make("PickPlaceSingle", n=6, seed=4)
    changed = 0
    for r in range(4):
        sel0, q0 = env.object_id.clone(), env.sim.qpos.clone()
        mask = torch.tensor([r % 2 == 0, True, False, r % 2 == 1, False, True])
        env.reset(mask)
        draw = env._sel_draw.to(torch.int32)
        assert torch.equal(env.object_id[~mask], sel0[~mask]) and torch.equal(env.sim.qpos[~mask], q0[~mask])
        assert torch.equal(env.object_id[mask], draw[mask])
        changed += int((env.object_id[mask] != sel0[mask]).sum())
    assert changed > 0


@pytest.mark.parametrize("task", ["PickPlaceSingle", "NutAssemblySingle"])
def test_selected_rows_are_the_selected_body_pose(task):
    env = _make(task, n=4, seed=2)
    key = "obj" if task.startswith("Pick") else "nut"
    names = env.obj_names if key == "obj" else env.nut_names
    for step in range(3):
        obs = env._get_observations()
        for e in range(4):
            k = int(env.object_id[e])
            o = env.sim.o[e]
            b = env.obj_body_id[names[k]]
            assert np.array_equal(obs[key + "_pos"][e].numpy(), o.xpos[b])
            assert np.array_equal(obs[key + "_quat"][e].numpy(), o.xquat[b][[1, 2, 3, 0]])
            assert float(obs[key + "_id"][e]) == k
        env.step(_actions(env, 1, step)[0])
    assert int(env.sim.warn.abs().max()) == 0


def test_out_of_range_selection_zeroes_the_rows_and_sets_warn_512():
    assert 512 in SIM_WARN_BITS
    env = _make("PickPlaceSingle", n=3, seed=2)
    env.sim.obj_sel[1] = 7
    env.step(_actions(env, 1)[0])
    a, b = env._modality_slices["object-state"]
    assert torch.equal(env.sim.obs[1, a + 7:b], torch.zeros(b - a - 7, dtype=torch.float64))
    assert env.sim.warn.tolist() == [0, 512, 0]


# ---- reward and success, restated from pick_place.py / nut_assembly.py (staged_rewards, reward, _check_success)
def _pp_expected(env, mode, shaping=True, scale=1.0):
    t, bits = env.sim.task_vec.numpy(), env.sim.task_out[:, 5].numpy().astype(np.int64)
    b2, bs, tb = env.bin2_pos, env.bin_size, env.target_bin_placements
    rew, succ = [], []
    for e in range(env.num_envs):
        eef, pos = t[e, 0:3], [t[e, 3 + 3 * i:6 + 3 * i] for i in range(4)]
        inb = []
        for i, p in enumerate(pos):
            x0 = b2[0] - (bs[0] / 2 if i in (0, 2) else 0)
            y0 = b2[1] - (bs[1] / 2 if i < 2 else 0)
            inside = x0 < p[0] < x0 + bs[0] / 2 and y0 < p[1] < y0 + bs[1] / 2 and b2[2] < p[2] < b2[2] + 0.1
            inb.append(inside and 1 - math.tanh(10 * np.linalg.norm(eef - p)) < 0.6)
        r = float(sum(inb))
        if shaping:
            act = [i for i in range(4) if not inb[i]]
            reach = grasp = lift = hover = 0.0
            if act:
                reach = (1 - math.tanh(10 * min(np.linalg.norm(pos[i] - eef) for i in act))) * 0.1
                grasp = 0.35 if any((bits[e] >> i) & 1 for i in act) else 0.0
                if grasp:
                    lift = 0.35 + (1 - math.tanh(15 * min(max(b2[2] + 0.25 - pos[i][2], 0.0) for i in act))) * 0.15
                hs = []
                for i in act:
                    d = math.hypot(pos[i][0] - tb[i, 0], pos[i][1] - tb[i, 1])
                    above = abs(pos[i][0] - tb[i, 0]) < bs[0] / 4 and abs(pos[i][1] - tb[i, 1]) < bs[1] / 4
                    hs.append((0.5 if above else lift) + (1 - math.tanh(10 * d)) * 0.2)
                hover = max(hs)
            r += max(reach, grasp, lift, hover)
        r *= scale
        if mode == 0:
            r /= 4.0
        rew.append(r)
        succ.append(sum(inb) > 0 if mode > 0 else sum(inb) == 4)
    return np.array(rew), np.array(succ)


def _nut_expected(env, mode, shaping=True, scale=1.0):
    t, bits = env.sim.task_vec.numpy(), env.sim.task_out[:, 5].numpy().astype(np.int64)
    rew, succ = [], []
    for e in range(env.num_envs):
        eef = t[e, 0:3]
        pos = [t[e, 3 + 6 * i:6 + 6 * i] for i in range(2)]
        handle = [t[e, 6 + 6 * i:9 + 6 * i] for i in range(2)]
        on = [abs(p[0] - env.peg_xy[i][0]) < 0.03 and abs(p[1] - env.peg_xy[i][1]) < 0.03 and p[2] < env.table_offset[2] + 0.05
              and 1 - math.tanh(10 * np.linalg.norm(eef - p)) < 0.6 for i, p in enumerate(pos)]
        r = float(sum(on))
        if shaping:
            act = [i for i in range(2) if not on[i]]
            reach = grasp = lift = hover = 0.0
            if act:
                reach = (1 - math.tanh(10 * min(np.linalg.norm(handle[i] - eef) for i in act))) * 0.1
                grasp = 0.35 if any((bits[e] >> i) & 1 for i in act) else 0.0
                if grasp:
                    lift = 0.35 + (1 - math.tanh(15 * min(max(env.table_z + 0.2 - pos[i][2], 0.0) for i in act))) * 0.15
                hover = max(lift + (1 - math.tanh(10 * np.linalg.norm(env.peg_xy[i] - pos[i][:2]))) * 0.2 for i in act)
            r += max(reach, grasp, lift, hover)
        r *= scale
        if mode == 0:
            r /= 2.0
        rew.append(r)
        succ.append(sum(on) > 0 if mode > 0 else sum(on) == 2)
    return np.array(rew), np.array(succ)


CASES = [("PickPlace", 0), ("PickPlaceCan", 2), ("PickPlaceSingle", 1), ("NutAssembly", 0), ("NutAssemblyRound", 2),
         ("NutAssemblySingle", 1)]


@pytest.mark.parametrize("task, mode", CASES)
def test_reward_and_success_follow_the_rules_over_a_rollout(task, mode):
    env = _make(task, n=3, seed=6, reward_shaping=True, reward_scale=2.0)
    expect = _pp_expected if task.startswith("Pick") else _nut_expected
    for a in _actions(env, 3, 1):
        _, r, _, _ = env.step(a)
        er, es = expect(env, mode, scale=2.0)
        assert np.allclose(r.numpy(), er, rtol=0, atol=1e-12), (r, er)
        assert np.array_equal(env._check_success().numpy(), es)


def _place(env, q, name, xyz):
    a = env.obj_qadr[name]
    q[:, a:a + 7] = torch.tensor([*xyz, 1.0, 0, 0, 0], dtype=q.dtype)


@pytest.mark.parametrize("task, mode", [c for c in CASES if c[0].startswith("Pick")])
def test_pickplace_hand_set_states(task, mode):
    """one object in its bin (success in modes 1 / 2, reward 1 + shaping, not divided by 4), a parked object (staged rewards still
    consider it), a grasp flag on a parked object"""
    env = _make(task, n=2, seed=3, reward_shaping=True)
    q = env.sim.qpos.clone()
    tb = env.target_bin_placements
    k = 3 if mode == 2 else int(env.object_id[0]) if mode == 1 else 0
    _place(env, q, env.obj_names[k], (tb[k, 0], tb[k, 1], env.bin2_pos[2] + 0.05))
    env.reset_to(q)
    if mode == 1:
        assert int(env.object_id[0]) == k  # reset_to keeps the selection
    r = env.reward().numpy()
    er, es = _pp_expected(env, mode)
    assert np.allclose(r, er, atol=1e-12) and np.array_equal(env._check_success().numpy(), es)
    assert bool(env.objects_in_bins[0, k])
    assert bool(es[0]) == (mode > 0)
    assert r[0] >= (1.0 if mode > 0 else 0.25)
    # grasp flag on every object (task_out[:, 5] as the grasp check writes it): parked objects count while not in their bins
    env.sim.task_out[:, 5] = 15.0
    r2 = env.reward().numpy()
    er2, _ = _pp_expected(env, mode)
    assert np.allclose(r2, er2, atol=1e-12) and (r2 >= r - 1e-12).all()


@pytest.mark.parametrize("task, mode", [c for c in CASES if c[0].startswith("Nut")])
def test_nut_hand_set_states(task, mode):
    env = _make(task, n=2, seed=3, reward_shaping=True)
    q = env.sim.qpos.clone()
    k = 1 if mode == 2 else int(env.object_id[0]) if mode == 1 else 0
    name = env.nut_names[k]
    # the nut's body frame over its peg, resting low on the table (the peg test reads the body position)
    _place(env, q, name, (env.peg_xy[k][0], env.peg_xy[k][1], env.table_offset[2] + 0.01))
    env.reset_to(q)
    r = env.reward().numpy()
    er, es = _nut_expected(env, mode)
    assert np.allclose(r, er, atol=1e-12) and np.array_equal(env._check_success().numpy(), es)
    assert bool(env.objects_on_pegs[0, k])
    env.sim.task_out[:, 5] = 3.0
    r2 = env.reward().numpy()
    er2, _ = _nut_expected(env, mode)
    assert np.allclose(r2, er2, atol=1e-12)


@pytest.mark.parametrize("task, kw", [
    ("PickPlace", dict(single_object_mode=2)),
    ("PickPlace", dict(single_object_mode=2, object_type="apple")),
    ("PickPlace", dict(object_type="Can")),
    ("PickPlace", dict(single_object_mode=3)),
    ("PickPlaceCan", dict(object_type="can")),
    ("PickPlaceMilk", dict(single_object_mode=2)),
    ("PickPlaceSingle", dict(single_object_mode=1)),
    ("NutAssembly", dict(single_object_mode=2)),
    ("NutAssembly", dict(single_object_mode=2, nut_type="hex")),
    ("NutAssemblySingle", dict(nut_type="round")),
    ("NutAssemblyRound", dict(nut_type="square")),
])
def test_wrong_keyword_combinations_raise(task, kw):
    with pytest.raises(ValueError):
        _make(task, **kw)
