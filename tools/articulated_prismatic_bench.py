"""Cost of prismatic joints on articulated robots: the prismatic step kernel (agx_hp1_articulated_step_prismatic, no IMU, no effort
DOF, no joint forces) on base_quadrotor_with_sliding_payload, and the same kernel against the plain one (agx_hp1_articulated_step)
on morphy_compliant and base_quadrotor_with_gimbal_camera, which have no prismatic joint (prismatic_mask 0): the cost of reading the
joint kinds at run time.  One physics sub-step per launch, timed with CUDA events over blocks of many launches, the kernels
alternating block by block in the same run.  The card's name and power limit are read in the same run.  One JSON line per run.

python tools/articulated_prismatic_bench.py [--envs 8192 65536] [--launches 200] [--blocks 7] [--out FILE]"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from tools.articulated_imu_bench import _sim_env, alternate  # noqa: E402
from tools.contact_bench import card  # noqa: E402

SHIPPED = "base_quadrotor_with_sliding_payload"
REVOLUTE = ("morphy_compliant", "base_quadrotor_with_gimbal_camera")


def engine(robot, n):
    import aerial_gym_simulator_b200.robots  # noqa: F401
    from aerial_gym_simulator_b200.config.env_config import EmptyEnvCfg
    from aerial_gym_simulator_b200.hp1 import Hp1Engine
    from aerial_gym_simulator_b200.registry._core import robot_registry

    r, _ = robot_registry.make_robot(robot, "lee_attitude_control", EmptyEnvCfg, "cuda:0")
    return Hp1Engine(r.make_spec(*_sim_env()), n, "cuda:0", articulation=r.make_articulation())


def prismatic_step(eng, act):
    """one launch of agx_hp1_articulated_step_prismatic on the engine's state, whatever its joint kinds"""
    from aerial_gym_simulator_b200 import _lib
    eng.physics_step(act, physics_steps=0)  # sets the buffers' actions and inputs (a no-op launch of the engine's own entry)
    eng.cfg.physics_steps = 1

    def run():
        _lib.check(eng.lib.agx_hp1_articulated_step_prismatic(eng._cfg_ref, eng._buf_ref, eng._art_ref, eng._prismatic, None, 0, None,
                                                              None, None, eng._stream()), "agx_hp1_articulated_step_prismatic")
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, nargs="+", default=[8192, 65536])
    ap.add_argument("--launches", type=int, default=200, help="kernel launches per timed block")
    ap.add_argument("--blocks", type=int, default=7, help="timed blocks per variant, alternating")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("articulated_prismatic_bench needs a CUDA device")
    name, power = card()
    out = {"tool": "articulated_prismatic_bench", "gpu": name, "power_limit": power, "launches_per_block": a.launches,
           "blocks": a.blocks, "kernel": {}}
    for n in a.envs:
        eng = engine(SHIPPED, n)
        act = torch.zeros(n, 4, device="cuda:0")
        assert eng._art_step_args()[0] == "agx_hp1_articulated_step_prismatic"
        med, times = alternate({"prismatic": lambda: eng.physics_step(act, physics_steps=1)}, a.launches, a.blocks)
        out["kernel"][f"{SHIPPED}/{n}"] = {"bodies": int(eng.body_state.shape[1]), "prismatic_us": round(med["prismatic"], 2),
                                           "prismatic_us_blocks": [round(x, 2) for x in times["prismatic"]]}
        del eng
        for robot in REVOLUTE:
            plain, pr = engine(robot, n), engine(robot, n)
            run = prismatic_step(pr, act)
            med, times = alternate({"plain": lambda: plain.physics_step(act, physics_steps=1), "prismatic": run}, a.launches, a.blocks)
            out["kernel"][f"{robot}/{n}"] = {"bodies": int(plain.body_state.shape[1]), "plain_us": round(med["plain"], 2),
                                             "prismatic_us": round(med["prismatic"], 2),
                                             "prismatic_over_plain": round(med["prismatic"] / med["plain"], 4),
                                             "plain_us_blocks": [round(x, 2) for x in times["plain"]],
                                             "prismatic_us_blocks": [round(x, 2) for x in times["prismatic"]]}
            del plain, pr
        torch.cuda.empty_cache()
    s = json.dumps(out)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
