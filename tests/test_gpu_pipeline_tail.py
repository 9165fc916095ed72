"""The pipeline's tail launch runs both capacity tiers: after a block barrier, warps of the block re-run the block's environments that
did not fit the small tier with the full-capacity layout (b2s_pipeline.cuh, tail_kernel), and it zeroes the group's work-list
counters for the next substep.  Only where and when the stages run changes, not their arithmetic: every case here is bit-identical
to the fused kernel over a contact-rich scripted Lift rollout (no GJK warm start, controller inside the tail)."""
import os

import numpy as np
import pytest

from tests.util import lift_states, load

pytestmark = pytest.mark.gpu


def _rollout(mode, nsub, substeps=300, n=16, precision="f32", tier_small=None, groups=None, poison=False):
    """`substeps` physics substeps as env_step calls of `nsub` substeps each -> (qpos, qvel, warn, time, launches of the calls)"""
    import torch
    from robosuite_b200 import controller_config as cc
    from robosuite_b200.engine import BatchedSim, CtrlCfg

    model = load("Lift_Panda")
    q, _ = lift_states(model, n, seed=21)
    calls = substeps // nsub
    rng = np.random.default_rng(3)
    actions = rng.uniform(-1, 1, size=(calls, n, 7))
    actions[:, :, 6] = 1.0  # keep closing the gripper: sliding / sticking finger contacts
    actions[calls // 4:, : (n + 1) // 2, :3] = [0.0, 0.0, -1.0]  # half of the arms (at least one) push down onto the table / cube
    os.environ["B2S_NO_GJK_CACHE"] = "1"
    os.environ["B2S_CTRL_SPLIT"] = "0"
    try:
        sim = BatchedSim(model, n, precision=precision, tier_small=tier_small)
        sim.ctrl_config(cc.resolve(model, cc.default_composite_config(), CtrlCfg))
        sim.set_export(False)
        if groups is not None:
            os.environ["B2S_GROUPS"] = str(groups)
        sim.set_mode(mode)  # reads B2S_GROUPS
    finally:
        os.environ.pop("B2S_GROUPS", None)
    dt = sim.dtype
    sim.qpos.copy_(torch.as_tensor(q, dtype=dt))
    sim.forward()
    sim.ctrl_reset()
    l0 = sim.launch_count
    for t in range(calls):
        if poison and t == calls // 2:
            # finite and below the divergence threshold (1e10) now, above it after one substep: the reset to the model defaults
            # happens in phase 0 of the call's SECOND substep
            sim.qpos[n // 2, 9] = 9.99e9
            sim.qvel[n // 2, 9] = 9e9
        sim.env_step(torch.as_tensor(actions[t], dtype=dt, device=sim.torch_device).contiguous(), nsub)
    torch.cuda.synchronize()
    launches = sim.launch_count - l0
    out = (sim.qpos.cpu().numpy().copy(), sim.qvel.cpu().numpy().copy(), sim.warn.cpu().numpy().copy(),
           sim.time.cpu().numpy().copy(), launches)
    sim.close()
    os.environ.pop("B2S_NO_GJK_CACHE", None)
    os.environ.pop("B2S_CTRL_SPLIT", None)
    return out


def _same(a, b):
    assert np.isfinite(b[0]).all()
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


@pytest.mark.parametrize("nsub", [1, 2, 3, 25])
def test_substeps_per_call_match_fused(nsub):
    """the counters zeroed by the tail serve the next substep inside a call; the head of every call zeroes them again"""
    a = _rollout(0, nsub)
    b = _rollout(1, nsub)
    _same(a, b)
    assert b[4] == (300 // nsub) * 8 * nsub * 3  # phase 0, phase 1 and the tail per substep and group


@pytest.mark.parametrize("groups", [None, 1])
def test_overflow_beyond_large_tier_warps_matches_fused(groups):
    """(4, 24): most environments overflow the small tier; in one group of 16 (one 16-warp Lift block) more per block than the
    block has full-capacity workspaces"""
    full = _rollout(1, 25)
    tier = _rollout(1, 25, tier_small=(4, 24), groups=groups)
    fused = _rollout(0, 25)
    _same(full, tier)
    _same(fused, tier)


@pytest.mark.parametrize("n,groups", [(1, None), (13, None), (16, 1)])
def test_group_shapes_match_fused(n, groups):
    """one environment; 13 in 8 uneven groups (a partly empty tail block); 16 in one group"""
    a = _rollout(0, 25, n=n)
    b = _rollout(1, 25, n=n, groups=groups)
    _same(a, b)


def test_f64_matches_fused():
    a = _rollout(0, 25, substeps=150, precision="f64")
    b = _rollout(1, 25, substeps=150, precision="f64")
    _same(a, b)


def test_divergence_reset_after_first_substep_matches_fused():
    """an environment that diverges during a call is reset by phase 0 of its next substep, in both schedules alike"""
    n = 16
    a = _rollout(0, 25, n=n, poison=True)
    b = _rollout(1, 25, n=n, poison=True)
    _same(a, b)
    assert int(b[2][n // 2]) & 32
    assert not (np.delete(b[2], n // 2) & 32).any()
    assert np.array_equal(a[3], b[3])
