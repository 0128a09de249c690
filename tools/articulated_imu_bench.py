"""Cost of the IMU on a link of an articulated robot:
  * the step kernel with the IMU input (agx_hp1_articulated_step_imu) against the plain one (agx_hp1_articulated_step), one physics
    sub-step per launch, for morphy_compliant (IMU on base_link) and base_quadrotor_with_gimbal_camera (IMU on gimbal_camera_link),
    timed with CUDA events over blocks of many launches, the two kernels alternating block by block in the same run;
  * the env step of EnvManager (empty_env, lee_attitude_control) for morphy_compliant against morphy_compliant_imu, the latter with
    render() -- the force-input glue and agx_imu_update -- after every step, alternating blocks of steps in the same run.
The card's name and power limit are read in the same run.  One JSON line per run.

python tools/articulated_imu_bench.py [--envs 8192 65536] [--launches 200] [--blocks 7] [--steps 50] [--out FILE]"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from tools.contact_bench import card  # noqa: E402

ROBOTS = {"morphy_compliant": ("morphy_compliant", "base_link"),
          "base_quadrotor_with_gimbal_camera": ("base_quadrotor_with_gimbal_camera", "gimbal_camera_link")}


def engines(robot, link, n):
    import aerial_gym_simulator_b200.robots  # noqa: F401
    from aerial_gym_simulator_b200.config.env_config import EmptyEnvCfg
    from aerial_gym_simulator_b200.hp1 import Hp1Engine
    from aerial_gym_simulator_b200.registry._core import robot_registry

    r, _ = robot_registry.make_robot(robot, "lee_attitude_control", EmptyEnvCfg, "cuda:0")
    spec, art = r.make_spec(*_sim_env()), r.make_articulation()
    plain = Hp1Engine(spec, n, "cuda:0", articulation=art)
    imu = Hp1Engine(spec, n, "cuda:0", articulation=art, imu_body=r.bodies.link_body[link])
    return plain, imu


def _sim_env():
    import aerial_gym_simulator_b200.env_manager  # noqa: F401  (registers the sim and env configs)
    from aerial_gym_simulator_b200.registry._core import env_config_registry, sim_config_registry
    return sim_config_registry.make_sim("base_sim"), env_config_registry.make_env("empty_env")


def timed(fn, reps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) * 1000.0 / reps


def alternate(fns, reps, blocks):
    for f in fns.values():
        timed(f, max(reps // 10, 1))  # warm-up
    times = {k: [] for k in fns}
    for _ in range(blocks):
        for k, f in fns.items():
            times[k].append(timed(f, reps))
    return {k: sorted(v)[len(v) // 2] for k, v in times.items()}, times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, nargs="+", default=[8192, 65536])
    ap.add_argument("--launches", type=int, default=200, help="kernel launches per timed block")
    ap.add_argument("--blocks", type=int, default=7, help="timed blocks per variant, alternating")
    ap.add_argument("--steps", type=int, default=50, help="env steps per timed block")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("articulated_imu_bench needs a CUDA device")
    name, power = card()
    out = {"tool": "articulated_imu_bench", "gpu": name, "power_limit": power, "launches_per_block": a.launches, "blocks": a.blocks,
           "kernel": {}, "env_step": {}}
    for robot, (r, link) in ROBOTS.items():
        for n in a.envs:
            plain, imu = engines(r, link, n)
            act = torch.zeros(n, 4, device="cuda:0")
            med, times = alternate({"plain": lambda: plain.physics_step(act, physics_steps=1),
                                    "imu": lambda: imu.physics_step(act, physics_steps=1)}, a.launches, a.blocks)
            out["kernel"][f"{robot}/{n}"] = {"imu_link": link, "plain_us": round(med["plain"], 2), "imu_us": round(med["imu"], 2),
                                             "imu_over_plain": round(med["imu"] / med["plain"], 4),
                                             "plain_us_blocks": [round(x, 2) for x in times["plain"]],
                                             "imu_us_blocks": [round(x, 2) for x in times["imu"]]}
            del plain, imu
            torch.cuda.empty_cache()
    from aerial_gym_simulator_b200.env_manager.env_manager import EnvManager
    for n in a.envs:
        envs = {k: EnvManager("base_sim", "empty_env", k, "lee_attitude_control", "cuda:0", num_envs=n, args={"seed": 0})
                for k in ("morphy_compliant", "morphy_compliant_imu")}
        for e in envs.values():
            e.reset()
        act = torch.zeros(n, 4, device="cuda:0")

        def plain():
            envs["morphy_compliant"].step(act)

        def with_imu():
            envs["morphy_compliant_imu"].step(act)
            envs["morphy_compliant_imu"].render()
        med, times = alternate({"plain": plain, "imu": with_imu}, a.steps, a.blocks)
        out["env_step"][str(n)] = {"morphy_compliant_us": round(med["plain"], 2), "morphy_compliant_imu_with_render_us": round(med["imu"], 2),
                                   "step_mode": envs["morphy_compliant_imu"].step_mode,
                                   "plain_us_blocks": [round(x, 2) for x in times["plain"]],
                                   "imu_us_blocks": [round(x, 2) for x in times["imu"]]}
        del envs
        torch.cuda.empty_cache()
    s = json.dumps(out)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
