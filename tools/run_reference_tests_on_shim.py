"""Run the REFERENCE'S OWN test functions (unmodified files under $ROBOSUITE_REFERENCE/tests) with the unmodified reference package on the
CPU oracle through oracle/mujoco_shim.  usage: python tools/run_reference_tests_on_shim.py [name ...]"""
import importlib.util
import os
import sys
import time
import traceback

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gen_env_golden as g  # noqa: E402

g.install()
REF = os.path.join(os.environ.get("ROBOSUITE_REFERENCE", ""), "tests")
TESTS = {
    "playback": ("test_environments/test_action_playback.py", "test_playback"),
    "panda_gripper": ("test_grippers/test_panda_gripper.py", "test_panda_gripper"),
    "rethink_gripper": ("test_grippers/test_rethink_gripper.py", None),
    "all_grippers": ("test_grippers/test_all_grippers.py", None),
    "robotiq_85": ("test_grippers/test_robotiq_85.py", None),
    "robotiq_140": ("test_grippers/test_robotiq_140.py", None),
    "robotiq_three": ("test_grippers/test_robotiq_threefinger.py", None),
    "jaco_three": ("test_grippers/test_jaco_threefinger.py", None),
    "all_robots": ("test_robots/test_all_robots.py", None),
    "composite_controllers": ("test_controllers/test_composite_controllers.py", None),
    "variable_impedance": ("test_controllers/test_variable_impedance.py", None),
    "linear_interpolator": ("test_controllers/test_linear_interpolator.py", None),
}


def load(path):
    spec = importlib.util.spec_from_file_location("ref_" + os.path.basename(path)[:-3], os.path.join(REF, path))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def composite(results):
    """test_composite_controllers.py is parametrised over every robot of the reference; the fixed-base single arms are this repo's scope"""
    mod = load("test_controllers/test_composite_controllers.py")
    for robot in ("Panda", "Sawyer", "IIWA", "UR5e", "Kinova3"):
        for ctrl in (None, "BASIC"):
            key = "composite_controllers::test_basic_controller_predefined_robots[%s-%s]" % (robot, ctrl)
            t0 = time.time()
            try:
                mod.test_basic_controller_predefined_robots.__wrapped__(robot, ctrl) if hasattr(mod.test_basic_controller_predefined_robots, "__wrapped__") \
                    else mod.test_basic_controller_predefined_robots(robot, ctrl)
                results[key] = ("passed", time.time() - t0)
            except Exception as e:  # noqa: BLE001
                traceback.print_exc()
                results[key] = ("FAILED %r" % (e,), time.time() - t0)


def main(names):
    results = {}
    for nm in names:
        if nm == "composite_controllers":
            composite(results)
            continue
        path, fn = TESTS[nm]
        mod = load(path)
        fns = [fn] if fn else [k for k in dir(mod) if k.startswith("test_")]
        for f in fns:
            t0 = time.time()
            try:
                getattr(mod, f)()
                results[nm + "::" + f] = ("passed", time.time() - t0)
            except Exception as e:  # noqa: BLE001
                traceback.print_exc()
                results[nm + "::" + f] = ("FAILED %r" % (e,), time.time() - t0)
    for k, (st, dt) in results.items():
        print("%-60s %s (%.1f s)" % (k, st, dt))
    return results


if __name__ == "__main__":
    names = sys.argv[1:] or list(TESTS)
    sys.argv = sys.argv[:1]  # some of the reference's test modules parse the command line at import time
    main(names)
