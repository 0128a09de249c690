"""Cost of contact between free obstacles: env-step time with dynamic obstacles and their ground contact
(args['contact_dynamic_obstacles'] = args['contact_obstacle_ground'] = True) and with obstacle-obstacle contact as well
(args['contact_obstacle_obstacle'] = True: one agx_obstacle_obstacle_contact launch after each sub-step's ground solve), and the
kernel alone, one JSON line.

Workload: dynamic_env (40 free-floating objects and the ground plane), lmf2 with velocity control, 8192 envs, 10 physics sub-steps
per env step (the env's own setting), graph step mode, random actions and random obstacle twists of up to 2 m/s (and 2 rad/s), with
every fifth env step without env_actions.  The two envs are built side by side and timed in alternating blocks of steps in the same
run, so both see the same card state.  Each block is timed with CUDA events; the line reports the median block.  The kernel alone is
timed with CUDA events over many launches on a copy of the rows the env with the key holds after the run.  The card's name and
power limit are read in the same run.

python tools/contact_obstacle_bench.py [--envs 8192] [--steps 50] [--blocks 10] [--launches 2000] [--out FILE]"""
import argparse
import json
import os
import random
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from tools.contact_bench import card  # noqa: E402


def make(pairs, n, seed=0):
    import aerial_gym_simulator_b200.task  # noqa: F401
    from aerial_gym_simulator_b200.sim import SimBuilder

    random.seed(seed)
    torch.manual_seed(seed)
    env = SimBuilder().build_env("base_sim", "dynamic_env", "lmf2", "lmf2_velocity_control", "cuda:0",
                                 args={"seed": seed, "contact": "rigid", "contact_moving_obstacles": True,
                                       "contact_dynamic_obstacles": True, "contact_obstacle_ground": True,
                                       "contact_obstacle_obstacle": pairs},
                                 num_envs=n, use_warp=True, headless=True)
    env.reset()
    return env


def kernel_time(env, launches):
    """mean time of one agx_obstacle_obstacle_contact launch on a copy of env's rows, us (the launches act on the copy in turn, as
    consecutive sub-steps would without the advance between them)"""
    from aerial_gym_simulator_b200.hp2 import ContactMotion, obstacle_obstacle_contact

    rows = env.global_tensor_dict["env_asset_state_tensor"].clone()
    args = (env.contact_params, ContactMotion(rows, env._obj_asset), env._obstacle_mass, env._obstacle_boxes)
    for _ in range(20):
        obstacle_obstacle_contact(*args)
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(launches):
        obstacle_obstacle_contact(*args)
    e.record()
    e.synchronize()
    return s.elapsed_time(e) * 1000.0 / launches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=8192)
    ap.add_argument("--steps", type=int, default=50, help="env steps per timed block")
    ap.add_argument("--blocks", type=int, default=10, help="timed blocks per mode, alternating")
    ap.add_argument("--launches", type=int, default=2000, help="launches of the kernel alone")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("contact_obstacle_bench needs a CUDA device")
    envs = {m: make(m, a.envs) for m in (False, True)}
    A = envs[False].num_obs_in_env
    g = torch.Generator(device="cuda:0").manual_seed(1)
    acts = [(torch.rand(a.envs, 4, generator=g, device="cuda:0") * 2 - 1) * 2.0 for _ in range(a.steps)]
    twists = []
    for s in range(a.steps):
        d = torch.randn(a.envs, A, 6, generator=g, device="cuda:0")
        d = d / d.view(a.envs, A, 2, 3).norm(dim=-1).repeat_interleave(3, dim=-1)
        tw = d * torch.rand(a.envs, A, 2, generator=g, device="cuda:0").repeat_interleave(3, dim=-1) * 2.0
        twists.append(None if s % 5 == 4 else tw)

    def block(env):
        for act, tw in zip(acts, twists):
            env.step(actions=act, **({} if tw is None else {"env_actions": tw}))
            env.reset_terminated_and_truncated_envs()

    for env in envs.values():  # warm-up: graph capture, module loads
        block(env)
    torch.cuda.synchronize()
    times = {m: [] for m in envs}
    for _ in range(a.blocks):
        for m, env in envs.items():
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            block(env)
            e.record()
            e.synchronize()
            times[m].append(s.elapsed_time(e) / a.steps)
    med = {m: sorted(t)[len(t) // 2] for m, t in times.items()}
    kern_us = kernel_time(envs[True], a.launches)
    name, power = card()
    ast = envs[True].global_tensor_dict["env_asset_state_tensor"]
    line = {
        "tool": "contact_obstacle_bench", "gpu": name, "power_limit": power, "envs": a.envs, "substeps_per_env_step": 10,
        "env": "dynamic_env", "robot": "lmf2", "obstacles": A, "max_twist": 2.0, "steps_without_env_actions": "every 5th",
        "steps_per_block": a.steps, "blocks": a.blocks,
        "ground_ms_per_env_step": round(med[False], 4), "pairs_ms_per_env_step": round(med[True], 4),
        "pairs_over_ground": round(med[True] / med[False], 3),
        "ground_ms_blocks": [round(t, 4) for t in times[False]], "pairs_ms_blocks": [round(t, 4) for t in times[True]],
        "kernel_us_per_launch": round(kern_us, 3), "kernel_launches": a.launches, "kernel_rows": int(ast.shape[0] * ast.shape[1]),
    }
    s = json.dumps(line)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
