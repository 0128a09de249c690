"""Cost of joint force sensing on articulated robots: the step kernel with the joint forces (agx_hp1_articulated_step_joint_force, no
IMU, no effort DOF) against the plain one (agx_hp1_articulated_step), one physics sub-step per launch, for morphy_compliant and
base_quadrotor_with_gimbal_camera, timed with CUDA events over blocks of many launches, the two kernels alternating block by block in
the same run.  The card's name and power limit are read in the same run.  The extra bytes each launch writes, (6 B + D) x 4 per env,
are reported beside the times.  One JSON line per run.

python tools/articulated_joint_force_bench.py [--envs 8192 65536] [--launches 200] [--blocks 7] [--out FILE]"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from tools.articulated_imu_bench import _sim_env, alternate  # noqa: E402
from tools.contact_bench import card  # noqa: E402

ROBOTS = ("morphy_compliant", "base_quadrotor_with_gimbal_camera")


def engines(robot, n):
    import aerial_gym_simulator_b200.robots  # noqa: F401
    from aerial_gym_simulator_b200.config.env_config import EmptyEnvCfg
    from aerial_gym_simulator_b200.hp1 import Hp1Engine
    from aerial_gym_simulator_b200.registry._core import robot_registry

    r, _ = robot_registry.make_robot(robot, "lee_attitude_control", EmptyEnvCfg, "cuda:0")
    spec, art = r.make_spec(*_sim_env()), r.make_articulation()
    return Hp1Engine(spec, n, "cuda:0", articulation=art), Hp1Engine(spec, n, "cuda:0", articulation=art, joint_force=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, nargs="+", default=[8192, 65536])
    ap.add_argument("--launches", type=int, default=200, help="kernel launches per timed block")
    ap.add_argument("--blocks", type=int, default=7, help="timed blocks per variant, alternating")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("articulated_joint_force_bench needs a CUDA device")
    name, power = card()
    out = {"tool": "articulated_joint_force_bench", "gpu": name, "power_limit": power, "launches_per_block": a.launches,
           "blocks": a.blocks, "kernel": {}}
    for robot in ROBOTS:
        for n in a.envs:
            plain, jf = engines(robot, n)
            act = torch.zeros(n, 4, device="cuda:0")
            med, times = alternate({"plain": lambda: plain.physics_step(act, physics_steps=1),
                                    "joint_force": lambda: jf.physics_step(act, physics_steps=1)}, a.launches, a.blocks)
            B, D = jf.joint_wrench.shape[1], jf.dof_force.shape[1]
            out["kernel"][f"{robot}/{n}"] = {"bodies": B, "extra_bytes": (6 * B + D) * 4 * n,
                                             "plain_us": round(med["plain"], 2), "joint_force_us": round(med["joint_force"], 2),
                                             "joint_force_over_plain": round(med["joint_force"] / med["plain"], 4),
                                             "plain_us_blocks": [round(x, 2) for x in times["plain"]],
                                             "joint_force_us_blocks": [round(x, 2) for x in times["joint_force"]]}
            del plain, jf
            torch.cuda.empty_cache()
    s = json.dumps(out)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
