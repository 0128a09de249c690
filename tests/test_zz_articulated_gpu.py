"""Articulated multirotors on the H100: agx_hp1_articulated_step against its host shadow, CUDA-graph step mode against launch mode,
the position task with morphy_compliant at scale, and the hover deflection on the device."""
import numpy as np
import pytest
import torch

from aerial_gym_simulator_b200.hp1 import Hp1Engine
from tests import _hp1_common as H
from tests._cpu_stack_articulated import CpuArticulatedHp1Engine, articulated_twin_for_dryrun
from tests.test_articulated_cpu import hover_check, morphy_compliant

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(autouse=True)
def _articulated_twin():
    """with --gpu-dryrun (tests/conftest.py has set DEV to "cpu" and entered the CPU stack) EnvManager and the engine below use the
    CPU twin that knows about joints; on the GPU nothing changes"""
    if DEV != "cpu":
        yield
        return
    with articulated_twin_for_dryrun():
        yield


def _engine(*a, **k):
    return Hp1Engine(*a, **k) if DEV != "cpu" else CpuArticulatedHp1Engine(*a, **k)


def test_kernel_matches_host_shadow():
    """4096 envs, random base states, joint states inside the limits, setpoints, thrusts, motor constants and actions, 10 sub-steps
    in one launch.  Tolerance: the kernel contracts multiply-adds into FMAs, the shadow does not (-ffp-contract=off), so results
    differ in the last bits and the 10 sub-steps of a closed-loop controller grow that; 5e-4 absolute on states of order 1 bounds it
    with margin.  An env whose joint lands within rounding of a limit can take the other branch of the projection: at most 0.1 %
    of the envs may exceed the tolerance, and every value must stay within 5e-2."""
    N = 4096 if DEV != "cpu" else 128
    _, art = morphy_compliant()
    spec = H.spec_from_registry("morphy_compliant", "lee_attitude_control")
    rng = np.random.default_rng(0)
    gpu = _engine(spec, N, DEV, per_env_params="all", articulation=art)
    cpu = CpuArticulatedHp1Engine(spec, N, per_env_params="all", articulation=art)
    root = np.zeros((N, 13), np.float32)
    root[:, 0:3] = rng.uniform(-3, 3, (N, 3))
    q = rng.normal(size=(N, 4))
    q[:, 0:2] *= 0.2
    root[:, 3:7] = q / np.linalg.norm(q, axis=1, keepdims=True)
    root[:, 7:13] = rng.uniform(-1, 1, (N, 6))
    dof = np.stack([rng.uniform(-0.5, 0.5, (N, 8)), rng.uniform(-2, 2, (N, 8))], axis=-1).astype(np.float32)
    vals = {"root_state": root, "dof_state": dof, "motor_thrust": rng.uniform(0.3, 1.2, (N, 4)),
            "dof_position_setpoint": rng.uniform(-0.3, 0.3, (N, 8)), "dof_velocity_setpoint": rng.uniform(-1, 1, (N, 8)),
            "tau_inc": rng.uniform(0.01, 0.03, (N, 4))}
    for e in (gpu, cpu):
        for k, v in vals.items():
            getattr(e, k).copy_(torch.tensor(np.asarray(v, np.float32)))
    act = torch.tensor(rng.uniform(-0.5, 0.5, (N, 4)), dtype=torch.float32)
    dist = torch.tensor(rng.uniform(-0.05, 0.05, (N, 6)), dtype=torch.float32)
    gpu.physics_step(act.to(DEV), disturbance=dist.to(DEV), physics_steps=10)
    cpu.physics_step(act, disturbance=dist, physics_steps=10)
    torch.cuda.synchronize()
    diffs = []
    for k in ("root_state", "dof_state", "motor_thrust"):
        g, c = getattr(gpu, k).cpu().reshape(N, -1), getattr(cpu, k).reshape(N, -1)
        assert torch.isfinite(g).all()
        diffs.append((g - c).abs().max(dim=1).values)
    per_env = torch.stack(diffs).max(dim=0).values
    assert per_env.max().item() < 5e-2, per_env.max().item()
    assert (per_env > 5e-4).float().mean().item() <= 1e-3, per_env.sort().values[-10:]


def _env(mode, n):
    from aerial_gym_simulator_b200.env_manager.env_manager import EnvManager
    torch.manual_seed(0)
    env = EnvManager("base_sim", "empty_env", "morphy_compliant", "lee_attitude_control", DEV, num_envs=n,
                     args={"step_mode": mode, "seed": 3})
    env.reset()
    return env


def test_graph_step_mode_is_bit_identical_to_launch_mode():
    n = 1024 if DEV != "cpu" else 64
    envs = {m: _env(m, n) for m in ("graph", "launch")}
    for env in envs.values():
        env.global_tensor_dict["dof_position_setpoint_tensor"].fill_(0.1)
    g = torch.Generator().manual_seed(1)
    for _ in range(20):
        a = (torch.rand(n, 4, generator=g) * 2 - 1) * 0.3
        for env in envs.values():
            env.step(a.to(DEV))
    torch.cuda.synchronize()
    gg, gl = envs["graph"].global_tensor_dict, envs["launch"].global_tensor_dict
    for k in ("robot_state_tensor", "dof_state_tensor", "robot_euler_angles"):
        assert torch.equal(gg[k], gl[k]), k
    assert torch.equal(envs["graph"].engine.motor_thrust, envs["launch"].engine.motor_thrust)
    if DEV != "cpu":
        assert envs["graph"].step_mode == "graph" and envs["graph"]._graphs


def test_position_task_at_scale(monkeypatch):
    from aerial_gym_simulator_b200.registry._core import task_registry
    import aerial_gym_simulator_b200.task  # noqa: F401
    N, steps = (65536, 520) if DEV != "cpu" else (256, 30)  # 520 > the 500-step episode: every env resets at least once
    monkeypatch.setattr(task_registry.get_task_config("position_setpoint_task"), "robot_name", "morphy_compliant")
    task = task_registry.make_task("position_setpoint_task", seed=2, num_envs=N, headless=True)
    task.reset()
    g = torch.Generator(device=DEV).manual_seed(0)
    gtd = task.sim_env.global_tensor_dict
    resets = 0
    for _ in range(steps):
        obs, rew, term, trunc, _ = task.step(torch.rand(N, 4, generator=g, device=DEV) * 2 - 1)
        resets += int((term | trunc).sum())
        q = gtd["dof_state_tensor"][..., 0]
        assert bool((q.abs() <= 0.6 + 1e-6).all())
    if DEV != "cpu":
        assert resets >= N
    for t in (obs["observations"], rew, gtd["robot_state_tensor"], gtd["dof_state_tensor"], task.sim_env.engine.motor_thrust):
        assert bool(torch.isfinite(t).all())
    if DEV != "cpu":
        task.sim_env.engine.check()
    task.close()


def test_hover_deflection_on_device():
    from aerial_gym_simulator_b200.env_manager.env_manager import EnvManager
    n = 64
    env = EnvManager("base_sim", "empty_env", "morphy_compliant", "lee_attitude_control", DEV, num_envs=n)
    env.spec.enable_disturbance = False
    env.reset()
    gtd = env.global_tensor_dict
    gtd["dof_state_tensor"].zero_()
    st = gtd["robot_state_tensor"]
    st[:, 3:13] = 0.0
    st[:, 6] = 1.0
    for _ in range(300):
        env.step(torch.zeros(n, 4, device=DEV))
    torch.cuda.synchronize()
    hover_check(env)
