#!/usr/bin/env python
"""Fly the three rigid-body rl_games checkpoints the reference ships (examples/rl_games_example/networks/*.pth, trained in Isaac Gym)
on this package's simulator and print a table: final hover error, crashes, per-episode return next to the checkpoint's own
`last_mean_rewards`.  Needs a reference checkout (AERIAL_GYM_REFERENCE).  --device cpu runs on the CPU twins of tests/_cpu_stack.py (host
shadow of the device code); --device cuda:0 on the real engine.

    python tools/fly_reference_policies.py [--device cpu] [--envs 256] > profiles/reference_policies_r1.md
"""
import argparse
import contextlib
import io
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
NETS = os.path.join(os.environ.get("AERIAL_GYM_REFERENCE", ""), "aerial_gym/examples/rl_games_example/networks")
CASES = [("position_setpoint_task", "attitude_policy.pth"), ("position_setpoint_task_sim2real", "vel_control_lmf2_direct.pth"),
         ("position_setpoint_task_acceleration_sim2real", "acc_command_2_multiplier_disturbance.pth")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--device", default="cpu")
    ap.add_argument("--envs", type=int, default=256)
    a = ap.parse_args()
    import aerial_gym_simulator_b200.task  # noqa: F401
    from aerial_gym_simulator_b200.registry._core import task_registry
    sys.path.insert(0, os.path.dirname(NETS))
    real_load = torch.load
    torch.load = lambda p, *x, **k: real_load(p, map_location=a.device, weights_only=False)
    from rl_games_inference import MLP
    if a.device == "cpu":
        from tests._cpu_stack import cpu_stack
        stack = cpu_stack()
    else:
        stack = contextlib.nullcontext()
    print("| task (robot, controller) | checkpoint | episodes | crashes | hover error at episode end: median / max [m] | mean return | "
          "checkpoint `last_mean_rewards` |\n|---|---|---|---|---|---|---|")
    with stack:
        for task_name, net in CASES:
            cfg = task_registry.get_task_config(task_name)
            cfg.device = a.device
            task = task_registry.make_task(task_name, seed=42, headless=True, num_envs=a.envs)
            task.reset()
            with contextlib.redirect_stdout(io.StringIO()):
                policy = MLP(cfg.observation_space_dim, cfg.action_space_dim, os.path.join(NETS, net)).to(a.device).eval()
            ck = real_load(os.path.join(NETS, net), map_location="cpu", weights_only=False)
            N, L = a.envs, cfg.episode_len_steps
            actions, ep, returns, crashes, last_dist = torch.zeros(N, cfg.action_space_dim, device=a.device), torch.zeros(N, device=a.device), [], 0, None
            with torch.no_grad():
                for i in range(2 * L + 2):
                    obs, rew, term, trunc, _ = task.step(actions)
                    ep += rew
                    done = term | trunc
                    crashes += int(term.sum())
                    if bool(done.any()):
                        returns += ep[done].tolist()
                        ep[done] = 0.0
                    else:
                        last_dist = (task.target_position - task.obs_dict["robot_position"]).norm(dim=1)
                    actions = policy(obs["observations"]).clamp(-1.0, 1.0).clone()  # rl_games clip_actions
            print(f"| `{task_name}` ({cfg.robot_name}, {cfg.controller_name}) | `{net}` | {len(returns)} | {crashes} | "
                  f"{float(last_dist.median()):.3f} / {float(last_dist.max()):.3f} | {np.mean(returns):.0f} | {float(ck['last_mean_rewards']):.0f} |")
            task.close()


if __name__ == "__main__":
    main()
