"""Cost of the rigid contact mode: env-step time in flag mode (geometric collision flag) and in contact mode (args['contact'] =
'rigid', agx_hp2_contact after every sub-step), one JSON line.

Workload: env_with_obstacles (panels, objects, six walls), lmf2 with velocity control, 8192 envs, 10 physics sub-steps per env step
(the env's own setting), graph step mode, random actions.  The two envs are built side by side and timed in alternating blocks of
steps in the same run, so both see the same card state.  Each block is timed with CUDA events; the line reports the median block.

python tools/contact_bench.py [--envs 8192] [--steps 50] [--blocks 10] [--out FILE]"""
import argparse
import json
import os
import random
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, power = (s.strip() for s in out.split(","))
        return name, power
    except Exception as e:  # the card name still comes from torch
        return torch.cuda.get_device_name(0), f"unknown ({e.__class__.__name__})"


def make(mode, n, seed=0):
    import aerial_gym_simulator_b200.task  # noqa: F401
    from aerial_gym_simulator_b200.sim import SimBuilder

    random.seed(seed)
    torch.manual_seed(seed)
    env = SimBuilder().build_env("base_sim", "env_with_obstacles", "lmf2", "lmf2_velocity_control", "cuda:0",
                                 args={"seed": seed, "contact": mode}, num_envs=n, use_warp=True, headless=True)
    env.reset()
    return env


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=8192)
    ap.add_argument("--steps", type=int, default=50, help="env steps per timed block")
    ap.add_argument("--blocks", type=int, default=10, help="timed blocks per mode, alternating")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("contact_bench needs a CUDA device")
    envs = {m: make(m, a.envs) for m in ("flag", "rigid")}
    g = torch.Generator(device="cuda:0").manual_seed(1)
    acts = [(torch.rand(a.envs, 4, generator=g, device="cuda:0") * 2 - 1) * 2.0 for _ in range(a.steps)]

    def block(env):
        for act in acts:
            env.step(actions=act)
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
    name, power = card()
    line = {
        "tool": "contact_bench", "gpu": name, "power_limit": power, "envs": a.envs, "substeps_per_env_step": 10,
        "env": "env_with_obstacles", "robot": "lmf2", "steps_per_block": a.steps, "blocks": a.blocks,
        "flag_ms_per_env_step": round(med["flag"], 4), "contact_ms_per_env_step": round(med["rigid"], 4),
        "contact_over_flag": round(med["rigid"] / med["flag"], 3),
        "flag_ms_blocks": [round(t, 4) for t in times["flag"]], "contact_ms_blocks": [round(t, 4) for t in times["rigid"]],
        "contact_crash_fraction_last_step": round(float(envs["rigid"].collision_tensor.float().mean()), 4),
    }
    s = json.dumps(line)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
