"""Time agx_hp1_articulated_body_state (articulated_body_state_kernel) with CUDA events, beside one sub-step of
agx_hp1_articulated_step in the same run, for morphy_compliant (B = 9) and base_quadrotor_with_gimbal_camera (B = 3) at 8,192 and
65,536 envs, and report each time against the HBM bound of the body-state pass: per env 52 B of root row + 8 D B of joint state read,
52 B B written, at 3.35 TB/s (the H100 SXM data sheet's figure for a 700 W card).

    python tools/articulated_body_state_bench.py [--iters 1000] [--out profiles/articulated_body_state_h100.json]

The card's name and power limit are read in the same run and stored beside the numbers."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12


def _gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip() if r.returncode == 0 else "nvidia-smi unavailable: " + r.stderr.strip()


def _time(fn, iters, warmup=50):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / iters  # us per launch


def run(robot, n, iters):
    from aerial_gym_simulator_b200.env_manager.env_manager import EnvManager
    torch.manual_seed(0)
    env = EnvManager("base_sim", "empty_env", robot, "lee_attitude_control", "cuda:0", num_envs=n, args={"seed": 0})
    env.spec.enable_disturbance = False
    env.reset()
    eng = env.engine
    B, D = eng.body_state.shape[1], eng.dof_state.shape[1]
    act = torch.zeros(n, 4, device="cuda:0")
    body_us = _time(eng.update_body_state, iters)
    step_us = _time(lambda: eng.physics_step(act, physics_steps=1), iters)
    eng.check()
    nbytes = n * (52 + 8 * D + 52 * B)
    bound_us = nbytes / HBM_BYTES_PER_S * 1e6
    return {"robot": robot, "num_envs": n, "bodies": B, "dofs": D, "iters": iters, "body_state_us": round(body_us, 2),
            "bytes": nbytes, "hbm_bound_us": round(bound_us, 2), "fraction_of_hbm_bound": round(bound_us / body_us, 3),
            "articulated_step_us_per_substep": round(step_us, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=1000)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "articulated_body_state_h100.json"))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    rows = [run(r, n, a.iters) for r in ("morphy_compliant", "base_quadrotor_with_gimbal_camera") for n in (8192, 65536)]
    res = {"gpu": _gpu_info(), "results": rows}
    print(json.dumps(res, indent=1))
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
