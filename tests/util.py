"""Shared helpers for the parity tests: build oracle + seeded Lift states."""
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# source checkout of the reference robosuite (v1.5.2): the tests that run the reference's own code skip without it
REFERENCE = os.environ.get("ROBOSUITE_REFERENCE", "")
PANDA_INIT = np.array([0, np.pi / 16.0, 0.00, -np.pi / 2.0 - np.pi / 3.0, 0.00, np.pi - 0.2, np.pi / 4])


def load(name="Lift_Panda"):
    from robosuite_b200.mjcf.compiler import load_model

    return load_model(os.path.join(ROOT, "tests", "golden", "models", name + ".npz"))


def lift_states(model, n, seed=0, vel=0.0):
    """Seeded reset-like states of Lift/Panda: arm at init pose + N(0,0.02^2) noise (robots/robot.py:247-259),
    gripper open, cube placed on the table with random xy / yaw (environments/manipulation/lift.py:311-336)."""
    rng = np.random.default_rng(seed)
    q = np.tile(model.qpos0, (n, 1))
    q[:, :7] = PANDA_INIT + rng.normal(0, 0.02, size=(n, 7))
    q[:, 7:9] = [0.020833, -0.020833]
    half_h = model.geom_size[model.names["geom"].index("cube_g0"), 2]
    q[:, 9] = rng.uniform(-0.03, 0.03, n)
    q[:, 10] = rng.uniform(-0.03, 0.03, n)
    q[:, 11] = 0.8 + 0.01 + half_h
    yaw = rng.uniform(0, 2 * np.pi, n)
    q[:, 12] = np.cos(yaw / 2)
    q[:, 13:15] = 0
    q[:, 15] = np.sin(yaw / 2)
    v = rng.normal(0, vel, size=(n, model.nv)) if vel > 0 else np.zeros((n, model.nv))
    return q, v


def dedegenerate_sawyer(model):
    """The composed Sawyer models carry two knife-edge coincidences that make constraint activation depend on the last bit of rounding
    in ANY engine: the l0 collision sphere exactly touches the rim of the base cylinder (dist = -5.6e-17 in fp64) and the gripper's
    initial qpos equals its joint limit.  Parity records that are to be replayed by more than one engine move both off the edge."""
    model.geom_size[model.names["geom"].index("robot0_link0_collision"), 0] -= 1e-5
    model.jnt_range[[model.names["joint"].index("gripper0_right_l_finger_joint"),
                     model.names["joint"].index("gripper0_right_r_finger_joint")]] += np.array([-1e-6, 1e-6])
    return model
