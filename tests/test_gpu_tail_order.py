"""The pipeline's tail hands its warps the group's environments in cost order when its blocks hold 8 warps or more (Lift f32: 16):
phase 0 files each environment under the cost class the tail wrote for it the substep before (`tail_key`), and each warp position of
the tail launch takes an environment by its rank, most expensive class first (b2s_pipeline.cuh, tail_env_at).  Which warp runs an
environment never changes its arithmetic: every case here is bit-identical to the fused kernel over the contact-rich scripted Lift
rollout, with many tail blocks per group."""
import numpy as np
import pytest

from tests.schedules import assert_same, lift_rollout, switches
from tests.util import lift_states, load

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n,groups,nsub,tier_small", [
    (256, 1, 25, None),       # 16 tail blocks in one group
    (1000, 8, 25, None),      # uneven groups, partial last blocks
    (256, 1, 1, None),        # the order of every substep comes from the previous call
    (256, 1, 25, (4, 24)),    # the first blocks get more overflowed environments than they have full-capacity warps
])
def test_ordered_tail_matches_fused(n, groups, nsub, tier_small):
    calls = 300 // nsub
    a = lift_rollout(0, calls, nsub, n=n, push_from=calls // 4)
    b = lift_rollout(1, calls, nsub, n=n, groups=groups, tier_small=tier_small, push_from=calls // 4)
    assert_same(a, b)


def test_ordered_tail_f64_matches_fused():
    """f64 Lift tail blocks hold fewer than 8 warps, below the sorting threshold of choose_blocks: the id-order tail kernel"""
    a = lift_rollout(0, 6, n=256, precision="f64", push_from=1)
    b = lift_rollout(1, 6, n=256, groups=1, precision="f64", push_from=1)
    assert_same(a, b)


def test_order_is_a_permutation_sorted_by_the_previous_keys():
    """after a call of one substep, the next call's tail runs every group's environments once each, ranked in non-increasing class
    of the keys the first call left"""
    import torch
    from robosuite_b200 import controller_config as cc
    from robosuite_b200.engine import BatchedSim, CtrlCfg

    n, G = 1000, 8
    model = load("Lift_Panda")
    q, _ = lift_states(model, n, seed=21)
    rng = np.random.default_rng(3)
    with switches(groups=G):
        sim = BatchedSim(model, n, precision="f32")
        sim.ctrl_config(cc.resolve(model, cc.default_composite_config(), CtrlCfg))
        sim.set_export(False)  # env_step runs the pipeline only without the derived-array export
        sim.set_mode(1)  # reads B2S_GROUPS
    sim.qpos.copy_(torch.as_tensor(q, dtype=sim.dtype))
    sim.forward()
    sim.ctrl_reset()

    def step(nsub, push):
        a = rng.uniform(-1, 1, size=(n, 7))
        a[:, 6] = 1.0
        if push:
            a[: n // 2, :3] = [0.0, 0.0, -1.0]
        sim.env_step(torch.as_tensor(a, dtype=sim.dtype, device=sim.torch_device).contiguous(), nsub)

    for t in range(8):
        step(25, t >= 2)
    step(1, True)
    torch.cuda.synchronize()
    key = sim.tail_key.cpu().numpy().copy()
    step(1, True)
    torch.cuda.synchronize()
    order = sim.tail_order.cpu().numpy()
    sim.close()
    assert len(np.unique(key)) > 1  # the rollout gives the environments different classes
    solo = 2  # TAIL_SOLO (b2s_types.cuh)

    def ranked(o, wpb):
        # rank of each warp position: the first `solo` blocks hold rank b in warp 0 and the cheapest ranks in their other warps
        m = len(o)
        rank = np.array([p - solo * (wpb - 1) if p // wpb >= solo else
                         (p // wpb if p % wpb == 0 else m - 1 - ((p // wpb) * (wpb - 1) + p % wpb - 1)) for p in range(m)])
        assert np.array_equal(np.sort(rank), np.arange(m))
        by_rank = np.empty(m, dtype=np.int64)
        by_rank[rank] = o
        return by_rank

    for g in range(G):
        e0, e1 = n * g // G, n * (g + 1) // G
        o = order[e0:e1]
        assert np.array_equal(np.sort(o), np.arange(e0, e1))
        # the model's tail block shape (8 to 16 warps when sorted, choose_blocks) is not exported: one of them must explain the order
        assert any((np.diff(key[ranked(o, w)]) <= 0).all() for w in range(8, 17))
