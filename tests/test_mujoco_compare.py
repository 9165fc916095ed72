"""tools/compare_with_mujoco.py: the direct oracle-vs-MuJoCo check.  Without a real MuJoCo installed the real comparison skips
itself; the script's plumbing (MJCF rewrite, constant comparison, state / control script, gating) is exercised against
`oracle/mujoco_shim` (the oracle behind mujoco's API), where every difference must be exactly zero."""
import importlib
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests.util import REFERENCE  # noqa: E402

REF_ASSETS = os.path.join(REFERENCE, "robosuite", "models", "assets") if REFERENCE else ""


def _tool():
    from tools import compare_with_mujoco

    return compare_with_mujoco


def test_helpers_are_deterministic_and_shaped():
    from tests.util import load

    t = _tool()
    m = load("Lift_Panda")
    q1, q2 = t.seeded_state(m, 3), t.seeded_state(m, 3)
    assert np.array_equal(q1, q2) and q1.shape == (m.nq,)
    assert not np.array_equal(q1, np.asarray(m.qpos0))
    assert np.array_equal(q1[9:], np.asarray(m.qpos0)[9:])  # only the robot joints are perturbed
    s = t.torque_script(m.nu, 7, 400, 0)
    assert s.shape == (400, m.nu) and np.abs(s[:, :7]).max() <= 4.0
    assert set(np.unique(s[:, 7:])) == {-1.0, 1.0}
    xml = t.load_mjcf("Lift_Panda", "/somewhere/assets")
    assert t.REF_ASSET_PREFIX not in xml and "<texture" not in xml and "/somewhere/assets/robots/panda/meshes/link0.stl" in xml


def _real_mujoco():
    """the real package, not oracle/mujoco_shim (which other tests put on sys.path)"""
    saved = sys.modules.pop("mujoco", None)
    path = [p for p in sys.path if "mujoco_shim" not in p]
    old, sys.path = sys.path, path
    try:
        mod = importlib.import_module("mujoco")
        return None if "b2s" in getattr(mod, "__version__", "") else mod
    except ImportError:
        return None
    finally:
        sys.path = old
        if saved is not None:
            sys.modules["mujoco"] = saved
        else:
            sys.modules.pop("mujoco", None)


@pytest.mark.skipif(not REF_ASSETS or not os.path.isdir(REF_ASSETS), reason="needs the mesh files of a reference checkout: set ROBOSUITE_REFERENCE")
def test_tool_plumbing_against_the_shim_is_exactly_zero(monkeypatch, capsys):
    shim = os.path.join(ROOT, "oracle", "mujoco_shim")
    monkeypatch.syspath_prepend(shim)
    monkeypatch.delitem(sys.modules, "mujoco", raising=False)
    t = _tool()
    rc = t.main(["--assets", REF_ASSETS, "--tasks", "Lift_Panda", "--steps", "30", "--gate-steps", "30"])
    out = capsys.readouterr().out
    sys.modules.pop("mujoco", None)
    assert rc == 0, out
    import json

    r = json.loads(out)["results"][0]
    assert r["ok"] and r["gate"]["max_dq_oracle"] == 0.0 and r["gate"]["max_dv_oracle"] == 0.0
    assert all(v == 0.0 for k, v in r["constants_max_abs_diff"].items() if isinstance(v, float))


def test_against_real_mujoco(capsys):
    if _real_mujoco() is None:
        pytest.skip("mujoco is not installed")
    assets = os.environ.get("B2S_ROBOSUITE_ASSETS")
    if assets is None:
        try:
            import robosuite

            assets = os.path.join(os.path.dirname(robosuite.__file__), "models", "assets")
        except ImportError:
            pytest.skip("set B2S_ROBOSUITE_ASSETS to robosuite/models/assets")
    sys.modules.pop("mujoco", None)
    rc = _tool().main(["--assets", assets, "--steps", "250"])
    assert rc == 0, capsys.readouterr().out
