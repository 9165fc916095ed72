"""The harness of the schedule comparisons: fused kernel (mode 0), phase pipeline (mode 1) and unit queue (mode 2) must give
bit-identical states.  libb2s has three test switches, environment variables it reads at fixed moments: B2S_GROUPS and
B2S_CTRL_SPLIT in b2s_set_mode, B2S_NO_GJK_CACHE at the first pipeline or unit-queue step.  Tests set them only through
`switches`, so a failing test cannot leave them set for the tests after it."""
import contextlib
import os
from collections import namedtuple

import numpy as np

from tests.util import lift_states, load


def _put(name, value):
    if value is None:
        os.environ.pop(name, None)
    else:
        os.environ[name] = value


@contextlib.contextmanager
def switches(gjk_cache=True, ctrl_split=True, groups=None):
    """B2S_NO_GJK_CACHE / B2S_CTRL_SPLIT / B2S_GROUPS as given (True / None: the variable absent, the library default) for the
    handles created, set_mode'd and first stepped inside; the previous values (absent or not) are restored on exit, also on error"""
    want = {"B2S_NO_GJK_CACHE": None if gjk_cache else "1", "B2S_CTRL_SPLIT": None if ctrl_split else "0",
            "B2S_GROUPS": None if groups is None else str(groups)}
    old = {k: os.environ.get(k) for k in want}
    try:
        for k, v in want.items():
            _put(k, v)
        yield
    finally:
        for k, v in old.items():
            _put(k, v)


def lift_actions(calls, n, seed=3, push_from=8, dim=7):
    """random arm actions with the gripper closing (sliding / sticking finger contacts exercise the friction cones); from call
    `push_from` on, half of the arms (at least one) push down onto the table / cube"""
    rng = np.random.default_rng(seed)
    a = rng.uniform(-1, 1, size=(calls, n, dim))
    a[:, :, dim - 1] = 1.0
    a[push_from:, : (n + 1) // 2, :3] = [0.0, 0.0, -1.0]
    return a


Rollout = namedtuple("Rollout", "qpos qvel warn time launches")


def lift_rollout(mode, calls, nsub=25, n=16, precision="f32", tier_small=None, groups=None, gjk_cache=False, ctrl_split=False,
                 push_from=8, poison=False, clean=False):
    """the contact-rich scripted Lift/Panda rollout: `calls` env_step calls of `nsub` substeps each from lift_states(seed 21) under
    lift_actions(push_from=push_from), run entirely inside switches(...).  The defaults are the settings under which the schedules
    are bit-identical: the fused kernel has no GJK warm start, and the pipeline's thread-per-environment OSC kernel orders its fp64
    sums differently from the controller inside the tail.  poison: environment n // 2 crosses the divergence threshold in
    the first substep of call calls // 2.  clean: no environment may set a warn bit.  Host copies of the final state, and the launches of the calls."""
    import torch
    from robosuite_b200 import controller_config as cc
    from robosuite_b200.engine import BatchedSim, CtrlCfg

    model = load("Lift_Panda")
    q, _ = lift_states(model, n, seed=21)
    actions = lift_actions(calls, n, push_from=push_from)
    with switches(gjk_cache, ctrl_split, groups):
        sim = BatchedSim(model, n, precision=precision, tier_small=tier_small)
        sim.ctrl_config(cc.resolve(model, cc.default_composite_config(), CtrlCfg))
        sim.set_export(False)
        sim.set_mode(mode)
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
    out = Rollout(sim.qpos.cpu().numpy().copy(), sim.qvel.cpu().numpy().copy(), sim.warn.cpu().numpy().copy(),
                  sim.time.cpu().numpy().copy(), sim.launch_count - l0)
    sim.close()
    if clean:
        assert int(np.abs(out.warn).max()) == 0
    return out


def assert_same(a, b):
    """two Rollouts: b's qpos finite, and bit-identical qpos and qvel"""
    assert np.isfinite(b.qpos).all()
    assert np.array_equal(a.qpos, b.qpos) and np.array_equal(a.qvel, b.qvel)


def make_env(task, n, mode, seed, groups=None, gjk_cache=True, ctrl_split=True, **make_kw):
    """suite.make(task, num_envs=n, seed=seed, **make_kw) switched to `mode`, both inside switches(...)"""
    import robosuite_b200 as suite

    with switches(gjk_cache, ctrl_split, groups):
        env = suite.make(task, num_envs=n, seed=seed, **make_kw)
        env.sim.set_mode(mode)
    return env


def random_actions(env, k, seed=0):
    """k steps of uniform actions in [-1, 1) from a seeded device generator"""
    import torch

    gen = torch.Generator(device=env.device)
    gen.manual_seed(seed)
    return torch.rand((k, env.num_envs, env.action_dim), generator=gen, device=env.device, dtype=env.dtype) * 2 - 1


def run(stepper, acts, fields=("qpos", "qvel", "obs")):
    """step `stepper` (an environment or a wrapper of one) through `acts`; clones of its sim's `fields` after the last step"""
    import torch

    for a in acts:
        stepper.step(a)
    torch.cuda.synchronize()
    return tuple(getattr(stepper.sim, f).clone() for f in fields)
