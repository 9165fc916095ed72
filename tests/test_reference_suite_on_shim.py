"""CPU, with a reference checkout in ROBOSUITE_REFERENCE only: the REFERENCE'S OWN test functions (unmodified files under its tests/, unmodified reference package) run
on the CPU oracle through oracle/mujoco_shim (tools/run_reference_tests_on_shim.py).  They are behavioural pins of the oracle's PHYSICS by
the reference's own acceptance criteria: bit-identical open-loop playback (test_action_playback.py), the gripper testers that must
close on a cube and lift it (test_panda_gripper.py, test_rethink_gripper.py, test_robotiq_*.py, test_jaco_threefinger.py,
test_all_grippers.py), and - slow, opt-in with B2S_REF_SLOW=1 - the
variable-impedance and linear-interpolator trajectory tests of the reference's OSC stack (test_variable_impedance.py,
test_linear_interpolator.py; 60 s each) and test_composite_controllers.py on the five fixed-base single arms (Panda, Sawyer, IIWA, UR5e,
Kinova3 x {None, BASIC}; 50 s); they passed when last run, DESIGN.md section 3)."""
import os
import subprocess
import sys

import pytest

from tests.util import REFERENCE, ROOT

pytestmark = pytest.mark.skipif(not REFERENCE or not os.path.isdir(os.path.join(REFERENCE, "tests")),
                                reason="needs a reference robosuite checkout: set ROBOSUITE_REFERENCE")


def _run(names, timeout):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "run_reference_tests_on_shim.py")] + names, capture_output=True, text=True,
                       timeout=timeout, cwd=ROOT)
    lines = [l for l in r.stdout.splitlines() if "::" in l]
    assert r.returncode == 0 and lines, r.stderr[-2000:]
    bad = [l for l in lines if "passed" not in l]
    assert not bad, bad
    return lines


def test_reference_playback_and_gripper_tests_pass_on_the_oracle():
    lines = _run(["playback", "panda_gripper", "rethink_gripper", "robotiq_85", "robotiq_140", "robotiq_three", "jaco_three", "all_grippers"], 600)
    assert len(lines) == 8


@pytest.mark.skipif(not os.environ.get("B2S_REF_SLOW"), reason="2 minutes: set B2S_REF_SLOW=1")
def test_reference_controller_trajectory_tests_pass_on_the_oracle():
    lines = _run(["variable_impedance", "linear_interpolator", "composite_controllers"], 1800)
    assert len(lines) == 12
