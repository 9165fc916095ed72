"""GPU: the step-1 export (b2s_set_step1_export, BatchedSim.set_step1_export, make(..., data_queries=True)) and the batched
MjData view (every schedule writing the full export's arrays: tests/test_gpu_exports.py).

* sim.data reads the poses the observations read;
* the errors."""
import pytest

from tests.schedules import make_env, random_actions

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu


def test_data_reads_the_poses_the_observations_read():
    env = make_env("Lift", 64, 1, 2, data_queries=True)
    d = env.sim.data
    acts = random_actions(env, 3, seed=4)
    for a in acts:
        obs, _, _, _ = env.step(a)
        assert torch.equal(obs["robot0_eef_pos"], d.get_site_xpos("gripper0_right_grip_site"))
        assert torch.equal(obs["cube_pos"], d.get_body_xpos("cube_main"))
        v = d.get_site_xvelp(env.eef_site_id)
        assert torch.equal(v, (d.get_site_jacp(env.eef_site_id) @ env.sim.qvel[:, :, None])[:, :, 0])
        assert torch.equal(d.full_m(), d.qM)
    env.close()


def test_errors():
    from robosuite_b200.engine import lib

    env = make_env("Lift", 2, 1, 0)
    env.step(torch.zeros((2, env.action_dim), device=env.device))
    for call in (lambda: env.sim.data.body_xpos, lambda: env.sim.data.get_site_jacp(0), lambda: env.sim.data.full_m()):
        with pytest.raises(RuntimeError, match="data_queries"):
            call()
    L = lib()
    assert L.b2s_set_step1_export(None, 1) == -1
    assert b"null handle" in L.b2s_last_error()
    assert L.b2s_set_step1_export(env.sim._h, 1) == 0 and L.b2s_set_step1_export(env.sim._h, 0) == 0
    env.close()
