"""Policies TRAINED IN THE REFERENCE (Isaac Gym / PhysX) flown on this package's integrator -- a behavioural check of SURVEY row a13
(the PhysX step, replaced here and "parity unpinned": no reference output can pin it).

The reference ships three rl_games checkpoints for rigid-body tasks under examples/rl_games_example/networks/ and the loader for them
(rl_games_inference.MLP, used unmodified).  Each one is run closed-loop, deterministic (mu), with rl_games' own action clamp to
[-1, 1] (its `clip_actions`, applied between network and env during training), on the task it was trained for, on the CPU twins:

    attitude_policy.pth                        position_setpoint_task                         base_quadrotor + lee_attitude_control
    vel_control_lmf2_direct.pth                position_setpoint_task_sim2real                lmf2 + lmf2_velocity_control
    acc_command_2_multiplier_disturbance.pth   position_setpoint_task_acceleration_sim2real   lmf2 + lmf2_acceleration_control

Bar: every env converges to its setpoint from the random reset state and holds it (no crash, no divergence); the per-episode return is
compared with the checkpoint's own `last_mean_rewards` for information only (the checkpoints predate the current reward functions).
Not a parity proof -- a controller tolerates model error -- but a wrong mass / inertia / thrust map / sign would show here.
Needs a reference checkout named by AERIAL_GYM_REFERENCE: skipped elsewhere."""
import contextlib
import io
import os
import sys

import pytest
import torch

NETS = os.path.join(os.environ.get("AERIAL_GYM_REFERENCE", ""), "aerial_gym/examples/rl_games_example/networks")
pytestmark = pytest.mark.skipif(not os.path.isdir(NETS), reason="reference checkout not present")

from ._cpu_stack import cpu_stack  # noqa: E402

CASES = [  # task, checkpoint, steps, steady-state distance bound [m]
    ("position_setpoint_task", "attitude_policy.pth", 450, 0.45),
    ("position_setpoint_task_sim2real", "vel_control_lmf2_direct.pth", 700, 0.25),
    ("position_setpoint_task_acceleration_sim2real", "acc_command_2_multiplier_disturbance.pth", 450, 0.35),
]


@pytest.mark.parametrize("task_name,net,steps,bound", CASES, ids=[c[0] for c in CASES])
def test_reference_trained_policy_flies_here(task_name, net, steps, bound, monkeypatch):
    import aerial_gym_simulator_b200.compat as compat
    import aerial_gym_simulator_b200.task  # noqa: F401
    from aerial_gym_simulator_b200.registry._core import task_registry
    compat.install()
    monkeypatch.setattr(task_registry.get_task_config(task_name), "device", "cpu")
    monkeypatch.syspath_prepend(os.path.dirname(NETS))
    real_load = torch.load
    monkeypatch.setattr(torch, "load", lambda p, *a, **k: real_load(p, map_location="cpu", weights_only=False))  # (the loader has no map_location)
    sys.modules.pop("rl_games_inference", None)
    from rl_games_inference import MLP  # the reference's loader, unmodified
    N = 96
    with cpu_stack():
        task = task_registry.make_task(task_name, seed=42, headless=True, num_envs=N)
        task.reset()
        with contextlib.redirect_stdout(io.StringIO()):
            policy = MLP(task.task_config.observation_space_dim, task.task_config.action_space_dim, os.path.join(NETS, net)).eval()
        actions = torch.zeros(N, task.task_config.action_space_dim)
        crashes, start = 0, None
        with torch.no_grad():
            for i in range(steps):
                obs, rew, term, trunc, _ = task.step(actions)
                crashes += int(term.sum())
                actions = policy(obs["observations"]).clamp(-1.0, 1.0).clone()
                dist = (task.target_position - task.obs_dict["robot_position"]).norm(dim=1)
                if i == 0:
                    start = dist.clone()
                assert torch.isfinite(obs["observations"]).all() and torch.isfinite(rew).all(), i
        assert steps < task.task_config.episode_len_steps and not bool(trunc.any())
    assert crashes == 0
    assert float(start.median()) > 0.6                                  # they start well away from the setpoint ...
    assert float(dist.max()) < bound and float(dist.median()) < 0.6 * bound, (float(dist.max()), float(dist.median()))  # ... and all arrive
    assert float(rew.mean()) > 9.0
