import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def _gpu_unavailable():
    """reason string when `gpu`-marked tests cannot run here, else None.  On a machine with a GPU a missing library is a FAILURE, not a skip
    (the product path has no CPU fallback and must fail loudly): only the absence of a CUDA device skips."""
    try:
        import torch

        if not torch.cuda.is_available():
            return "no CUDA device (these tests run on an H100: pytest -m gpu)"
    except Exception as e:  # pragma: no cover
        return "torch unavailable: %r" % (e,)
    return None


def pytest_collection_modifyitems(config, items):
    reason = _gpu_unavailable()
    if reason is None:
        return
    skip = pytest.mark.skip(reason=reason)
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def lift_model():
    from robosuite_b200.mjcf.compiler import load_model

    return load_model(os.path.join(ROOT, "tests", "golden", "models", "Lift_Panda.npz"))


@pytest.fixture(autouse=True)
def _close_handles():
    """A device holds at most 8 live handles (constant-memory descriptor slots): tests that fail, or simply do not close their
    simulators, must not starve the ones after them."""
    yield
    eng = sys.modules.get("robosuite_b200.engine")
    if eng is not None:
        eng.close_all()
