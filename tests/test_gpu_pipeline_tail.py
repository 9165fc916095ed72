"""The pipeline's tail launch runs both capacity tiers: after a block barrier, warps of the block re-run the block's environments that
did not fit the small tier with the full-capacity layout (b2s_pipeline.cuh, tail_kernel), and it zeroes the group's work-list
counters for the next substep.  Only where and when the stages run changes, not their arithmetic: every case here is bit-identical
to the fused kernel over a contact-rich scripted Lift rollout (no GJK warm start, controller inside the tail)."""
import numpy as np
import pytest

from tests.schedules import assert_same, lift_rollout

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("nsub", [1, 2, 3, 25])
def test_substeps_per_call_match_fused(nsub):
    """the counters zeroed by the tail serve the next substep inside a call; the head of every call zeroes them again"""
    calls = 300 // nsub
    a = lift_rollout(0, calls, nsub, push_from=calls // 4)
    b = lift_rollout(1, calls, nsub, push_from=calls // 4)
    assert_same(a, b)
    assert b.launches == calls * 8 * nsub * 3  # phase 0, phase 1 and the tail per substep and group


@pytest.mark.parametrize("groups", [None, 1])
def test_overflow_beyond_large_tier_warps_matches_fused(groups):
    """(4, 24): most environments overflow the small tier; in one group of 16 (one 16-warp Lift block) more per block than the
    block has full-capacity workspaces"""
    full = lift_rollout(1, 12, push_from=3)
    tier = lift_rollout(1, 12, tier_small=(4, 24), groups=groups, push_from=3)
    fused = lift_rollout(0, 12, push_from=3)
    assert_same(full, tier)
    assert_same(fused, tier)


@pytest.mark.parametrize("n,groups", [(1, None), (13, None), (16, 1)])
def test_group_shapes_match_fused(n, groups):
    """one environment; 13 in 8 uneven groups (a partly empty tail block: groups of 1 and 2); 16 in one group.  Every group's
    launch chain is one CUDA graph replayed on the group's own stream, one group included.  1000 substeps."""
    a = lift_rollout(0, 40, n=n, push_from=10)
    b = lift_rollout(1, 40, n=n, groups=groups, push_from=10)
    assert_same(a, b)


def test_f64_matches_fused():
    assert_same(lift_rollout(0, 6, precision="f64", push_from=1), lift_rollout(1, 6, precision="f64", push_from=1))


def test_divergence_reset_after_first_substep_matches_fused():
    """an environment that diverges during a call is reset by phase 0 of its next substep, in both schedules alike"""
    n = 16
    a = lift_rollout(0, 12, n=n, push_from=3, poison=True)
    b = lift_rollout(1, 12, n=n, push_from=3, poison=True)
    assert_same(a, b)
    assert int(b.warn[n // 2]) & 32
    assert not (np.delete(b.warn, n // 2) & 32).any()
    assert np.array_equal(a.time, b.time)
