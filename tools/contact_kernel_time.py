"""Time each contact kernel alone against another build of the library, one JSON line: A/B runs of a change to contact_core.cuh
or the contact kernels.

Inputs: 8192 envs (--envs) after warm-up env steps with random actions (and, in dynamic_env, random obstacle twists of up to 2 m/s
and 2 rad/s): env_with_obstacles in contact mode for agx_hp2_contact, and dynamic_env with moving, dynamic, obstacle-ground and
obstacle-obstacle contact for agx_hp2_contact_moving, agx_hp2_contact_dynamic, agx_obstacle_ground_contact and
agx_obstacle_obstacle_contact.  The state the kernels read and write (robot rows, asset rows, force, crash flags) is snapshot once.
Each block restores the snapshot, runs 10 untimed launches, then times --launches launches of one kernel with CUDA events (the
launches act on the state in turn, as consecutive sub-steps would without the rest of the step between them).  The two builds
alternate block by block, --rounds times each (ABAB...), and after every pair of blocks the state each left must be bit-identical.
The card's name and power limit are read in the same run.

python tools/contact_kernel_time.py --other-lib PATH [--envs 8192] [--launches 500] [--rounds 4] [--out FILE]

PATH is the other build's libaerial_gym_b200.so (same ABI), e.g. the parent commit's, reported as "other"; the tree's build is
"this"."""
import argparse
import json
import os
import random
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from tools.contact_bench import card  # noqa: E402


def make(env_name, args, n, seed=0):
    import aerial_gym_simulator_b200.task  # noqa: F401
    from aerial_gym_simulator_b200.sim import SimBuilder

    random.seed(seed)
    torch.manual_seed(seed)
    env = SimBuilder().build_env("base_sim", env_name, "lmf2", "lmf2_velocity_control", "cuda:0", args={"seed": seed, **args},
                                 num_envs=n, use_warp=True, headless=True)
    env.reset()
    return env


def warm_up(env, steps, twists):
    g = torch.Generator(device="cuda:0").manual_seed(1)
    E = env.num_envs
    for s in range(steps):
        act = (torch.rand(E, 4, generator=g, device="cuda:0") * 2 - 1) * 2.0
        kw = {}
        if twists and s % 5 != 4:
            A = env.num_obs_in_env
            d = torch.randn(E, A, 6, generator=g, device="cuda:0")
            d = d / d.view(E, A, 2, 3).norm(dim=-1).repeat_interleave(3, dim=-1)
            kw["env_actions"] = d * torch.rand(E, A, 2, generator=g, device="cuda:0").repeat_interleave(3, dim=-1) * 2.0
        env.step(actions=act, **kw)
        env.reset_terminated_and_truncated_envs()
    torch.cuda.synchronize()


def kernels(rigid, dyn):
    """name -> (launch, the tensors it reads and writes)"""
    from aerial_gym_simulator_b200 import hp2

    def robot(env, moving, dynamic):
        force, crashes = env.global_tensor_dict["robot_contact_force_tensor"], env.collision_tensor
        motion = env._contact_motion if moving else None
        mass = env._obstacle_mass if dynamic else None
        state = [env.engine.root_state, force, crashes] + ([motion.asset_state] if dynamic else [])
        return (lambda: hp2.contact(env.scene, env.engine.root_state, env.contact_params, force, crashes, motion=motion, mass=mass),
                state)

    rows = dyn._contact_motion.asset_state
    return {
        "hp2_contact_kernel": robot(rigid, False, False),
        "hp2_contact_moving_kernel": robot(dyn, True, False),
        "hp2_contact_dynamic_kernel": robot(dyn, True, True),
        "obstacle_ground_contact_kernel": (
            lambda: hp2.obstacle_ground_contact(dyn.contact_params, dyn._contact_motion, dyn._obstacle_mass, dyn._obstacle_hull), [rows]),
        "obstacle_obstacle_contact_kernel": (
            lambda: hp2.obstacle_obstacle_contact(dyn.contact_params, dyn._contact_motion, dyn._obstacle_mass, dyn._obstacle_boxes),
            [rows]),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--other-lib", required=True, help="the other build's libaerial_gym_b200.so")
    ap.add_argument("--envs", type=int, default=8192)
    ap.add_argument("--warmup-steps", type=int, default=30, help="env steps before the snapshot")
    ap.add_argument("--launches", type=int, default=500, help="timed launches per block")
    ap.add_argument("--rounds", type=int, default=4, help="blocks per build, alternating")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("contact_kernel_time needs a CUDA device")
    from aerial_gym_simulator_b200 import _lib

    rigid = make("env_with_obstacles", {"contact": "rigid"}, a.envs)
    dyn = make("dynamic_env", {"contact": "rigid", "contact_moving_obstacles": True, "contact_dynamic_obstacles": True,
                               "contact_obstacle_ground": True, "contact_obstacle_obstacle": True}, a.envs)
    warm_up(rigid, a.warmup_steps, False)
    warm_up(dyn, a.warmup_steps, True)
    # both builds typed by _lib.load(); the hp2 wrappers call whichever _lib._lib holds
    this = _lib.load()
    _lib._lib = None
    os.environ["AGX_LIB_PATH"] = os.path.abspath(a.other_lib)
    try:
        other = _lib.load()
    finally:
        del os.environ["AGX_LIB_PATH"]
        _lib._lib = this
    builds = {"other": other, "this": this}

    out = {"tool": "contact_kernel_time", "envs": a.envs, "launches_per_block": a.launches, "rounds": a.rounds, "kernels": {}}
    for name, (launch, state) in kernels(rigid, dyn).items():
        snap = [t.clone() for t in state]
        us = {b: [] for b in builds}
        for _ in range(a.rounds):
            left = {}
            for b, lib in builds.items():
                _lib._lib = lib
                for t, s in zip(state, snap):
                    t.copy_(s)
                for _ in range(10):
                    launch()
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                for _ in range(a.launches):
                    launch()
                e.record()
                e.synchronize()
                us[b].append(s.elapsed_time(e) * 1000.0 / a.launches)
                left[b] = [t.clone() for t in state]
            if not all(torch.equal(x, y) for x, y in zip(left["other"], left["this"])):
                raise SystemExit(f"{name}: the two builds left different state")
        _lib._lib = this
        med = {b: sorted(v)[len(v) // 2] for b, v in us.items()}
        out["kernels"][name] = {
            "us_per_launch_median": {b: round(m, 3) for b, m in med.items()},
            "this_over_other": round(med["this"] / med["other"], 4),
            "other_spread_us": round(max(us["other"]) - min(us["other"]), 3),
            "us_per_launch_blocks": {b: [round(t, 3) for t in v] for b, v in us.items()},
            "same_state": True,
        }
    out["gpu"], out["power_limit"] = card()
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
