"""The phase pipeline with a single live environment group, and with an uneven split into groups, against the fused kernel.
Every group's launch chain is one CUDA graph replayed on the group's own stream, one group included."""
import numpy as np
import pytest

from tests.test_gpu_engine import _scripted_rollout

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n, groups", [(1, None), (16, 1), (13, None)], ids=["n_env_1", "groups_1", "n_env_13"])
def test_pipeline_groups_match_fused_bit_exact(n, groups):
    """one environment, and 16 environments with B2S_GROUPS=1, run a single group; 13 environments in the default 8 groups give
    groups of 1 and 2 environments.  Without the GJK warm start and with the controller inside the tail kernel (the settings of
    test_pipeline_mode_matches_fused_bit_exact) each is bit-identical to the fused kernel over a contact-rich 1000-substep rollout."""
    a = _scripted_rollout(0, 40, True, n=n)
    b = _scripted_rollout(1, 40, True, n=n, groups=groups)
    assert np.isfinite(b[0]).all()
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
