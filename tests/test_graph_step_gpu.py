"""EnvManager.step as ONE CUDA-graph launch per env step (args['step_mode'] = 'graph', the default on CUDA with the device RNG) against the
launch-by-launch loop: same kernels, same in-kernel Philox draws, same collision flags -- trajectories must coincide bit for bit.  Also the
in-kernel disturbance draw of the HP1 physics launch against agx_disturbance_draw feeding the [N,6] buffer."""
import contextlib
import random

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _env(mode, robot, controller, seed=4, n=64):
    import aerial_gym_simulator_b200.task  # noqa: F401
    from aerial_gym_simulator_b200.sim import SimBuilder

    random.seed(seed)
    torch.manual_seed(seed)
    env = SimBuilder().build_env("base_sim", "env_with_obstacles", robot, controller, DEV, args={"seed": seed, "step_mode": mode},
                                 num_envs=n, use_warp=True, headless=True)
    env.reset()
    return env


@pytest.mark.parametrize("robot,controller", [("lmf2", "lmf2_velocity_control"), ("base_octarotor", "octarotor_velocity_control")])
def test_graph_step_equals_launch_loop(robot, controller):
    a, b = _env("graph", robot, controller), _env("launch", robot, controller)
    assert a.step_mode == ("graph" if DEV != "cpu" else "launch") and b.step_mode == "launch"  # no CUDA graph on the CPU twin
    assert torch.equal(a.engine.root_state, b.engine.root_state)
    g = torch.Generator(device=DEV).manual_seed(1)
    any_crash = False
    for step in range(12):
        act = torch.rand(a.num_envs, a.num_robot_actions, generator=g, device=DEV) * 2 - 1
        random.seed(100 + step)
        a.step(actions=act)
        random.seed(100 + step)
        b.step(actions=act)
        torch.cuda.synchronize()
        assert torch.equal(a.engine.root_state, b.engine.root_state), f"step {step}"
        assert torch.equal(a.engine.motor_thrust, b.engine.motor_thrust)
        assert torch.equal(a.collision_tensor, b.collision_tensor)
        assert torch.equal(a.engine.sim_steps, b.engine.sim_steps)
        any_crash |= bool(a.collision_tensor.any())
        if step == 5:  # a masked reset in between: the graph keeps working on the same buffers
            ids = torch.arange(0, a.num_envs, 3, device=DEV)
            random.seed(7); torch.manual_seed(7)
            a.reset_idx(ids)
            random.seed(7); torch.manual_seed(7)
            b.reset_idx(ids)
    assert (len(a._graphs) >= 1 or DEV == "cpu") and a._dist_counter == b._dist_counter
    if a.spec.enable_disturbance and DEV != "cpu":  # the device-side draw counter of graph mode
        assert int(a._dist_ctr_dev.item()) == a._dist_counter & 0xFFFFFFFF and a._dist_counter >= 100
    if DEV != "cpu":
        a.engine.check()


def test_in_kernel_disturbance_equals_separate_draw():
    """physics launch with AgxHp1Buffers.dist_counter (draw inside the kernel) == agx_disturbance_draw into [N,6] + the same launch"""
    _check_in_kernel_disturbance("base_octarotor", "octarotor_velocity_control")


def test_articulated_in_kernel_disturbance_equals_separate_draw():
    """the same for morphy_compliant: it takes the articulated step, whose kernel has its own copy of the in-kernel draw, and its
    joint state must agree bit for bit too"""
    _check_in_kernel_disturbance("morphy_compliant", "lee_attitude_control")


def _check_in_kernel_disturbance(robot, controller):
    import aerial_gym_simulator_b200.task  # noqa: F401
    from aerial_gym_simulator_b200.sim import SimBuilder
    from tests._cpu_stack_articulated import articulated_twin_for_dryrun

    with articulated_twin_for_dryrun() if DEV == "cpu" else contextlib.nullcontext():
        n = 513
        mk = lambda: SimBuilder().build_env("base_sim", "empty_env", robot, controller, DEV, args={"seed": 9}, num_envs=n, headless=True)
        e1, e2 = mk(), mk()
    articulated = e1.engine.dof_state is not None
    assert e1.spec.enable_disturbance and articulated == (robot == "morphy_compliant")
    for e in (e1, e2):
        torch.manual_seed(3)
        e.reset()
    assert torch.equal(e1.engine.root_state, e2.engine.root_state)

    def same():
        torch.cuda.synchronize()
        return torch.equal(e1.engine.root_state, e2.engine.root_state) and (
            not articulated or torch.equal(e1.engine.dof_state, e2.engine.dof_state))

    act = torch.rand(n, 4, device=DEV) * 2 - 1
    ctr = torch.tensor([0], dtype=torch.int32, device=DEV)
    differs = False
    for step in range(6):
        e1.engine.physics_step(act, disturbance=e1._draw_disturbance(), physics_steps=1)   # draw counter = step
        e2.engine.physics_step(act, physics_steps=1, dist_counter=ctr, dist_offset=step)  # *ctr + offset = step
        assert same(), f"step {step}"
        differs |= bool(e1._dist_buf.abs().sum() > 0)
    assert differs  # some env did receive a disturbance in six draws of 513 envs at p = 0.05..0.1
    # three fused sub-steps in ONE launch draw counters c, c+1, c+2
    e1.engine.physics_step(act, disturbance=e1._draw_disturbance(), physics_steps=1)
    e1.engine.physics_step(act, disturbance=e1._draw_disturbance(), physics_steps=1)
    e1.engine.physics_step(act, disturbance=e1._draw_disturbance(), physics_steps=1)
    ctr.fill_(6)
    e2.engine.physics_step(act, physics_steps=3, dist_counter=ctr, dist_offset=0)
    assert same()
