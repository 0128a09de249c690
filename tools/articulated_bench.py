"""Cost of the articulated step: median env step of position_setpoint_task (lee_attitude_control) for
  * morphy_compliant (agx_hp1_articulated_step on the task's un-fused path),
  * morphy_stiff on the same un-fused path (agx_hp1_physics_step, then the same host sequence),
  * morphy_stiff fused (one agx_hp1_position_task_step per env step), for context,
at each env count, timed in alternating blocks of steps in the same run so all three see the same card state (CUDA events around
each block; the median block is reported).  The physics kernels alone are timed with CUDA events over many launches of one physics
sub-step on the two engines.  The card's name and power limit are read in the same run.  One JSON line per run.

python tools/articulated_bench.py [--envs 8192 65536] [--steps 50] [--blocks 7] [--launches 500] [--out FILE]"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from tools.contact_bench import card  # noqa: E402


def make(robot, n, unfused):
    import aerial_gym_simulator_b200.task  # noqa: F401
    from aerial_gym_simulator_b200.registry._core import task_registry

    cfg = task_registry.get_task_config("position_setpoint_task")
    old = cfg.robot_name
    cfg.robot_name = robot
    try:
        task = task_registry.make_task("position_setpoint_task", seed=0, num_envs=n, headless=True)
    finally:
        cfg.robot_name = old
    task._unfused = task._unfused or unfused
    task.reset()
    return task


def kernel_us(task, launches):
    eng = task.sim_env.engine
    a = torch.zeros(eng.N, 4, device="cuda:0")
    keep = (eng.root_state.clone(), eng.motor_thrust.clone(), None if eng.dof_state is None else eng.dof_state.clone())
    for _ in range(20):
        eng.physics_step(a, physics_steps=1)
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(launches):
        eng.physics_step(a, physics_steps=1)
    e.record()
    e.synchronize()
    eng.root_state.copy_(keep[0]); eng.motor_thrust.copy_(keep[1])
    if keep[2] is not None:
        eng.dof_state.copy_(keep[2])
    return s.elapsed_time(e) * 1000.0 / launches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, nargs="+", default=[8192, 65536])
    ap.add_argument("--steps", type=int, default=50, help="env steps per timed block")
    ap.add_argument("--blocks", type=int, default=7, help="timed blocks per variant, alternating")
    ap.add_argument("--launches", type=int, default=500, help="launches of each physics kernel alone")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("articulated_bench needs a CUDA device")
    variants = {"morphy_compliant": ("morphy_compliant", True), "morphy_stiff_unfused": ("morphy_stiff", True),
                "morphy_stiff_fused": ("morphy_stiff", False)}
    name, power = card()
    out = {"tool": "articulated_bench", "gpu": name, "power_limit": power, "task": "position_setpoint_task",
           "controller": "lee_attitude_control", "steps_per_block": a.steps, "blocks": a.blocks, "sizes": {}}
    for n in a.envs:
        tasks = {k: make(r, n, u) for k, (r, u) in variants.items()}
        assert not tasks["morphy_stiff_fused"]._unfused and tasks["morphy_stiff_unfused"]._unfused
        g = torch.Generator(device="cuda:0").manual_seed(1)
        acts = [torch.rand(n, 4, generator=g, device="cuda:0") * 2 - 1 for _ in range(a.steps)]

        def block(task):
            for act in acts:
                task.step(act)

        for t in tasks.values():
            block(t)  # warm-up
        torch.cuda.synchronize()
        times = {k: [] for k in tasks}
        for _ in range(a.blocks):
            for k, t in tasks.items():
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                block(t)
                e.record()
                e.synchronize()
                times[k].append(s.elapsed_time(e) * 1000.0 / a.steps)
        med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
        r = {f"{k}_us_per_env_step": round(v, 2) for k, v in med.items()}
        r.update({f"{k}_us_blocks": [round(x, 2) for x in v] for k, v in times.items()})
        r["compliant_over_stiff_unfused"] = round(med["morphy_compliant"] / med["morphy_stiff_unfused"], 3)
        r["articulated_kernel_us_per_substep"] = round(kernel_us(tasks["morphy_compliant"], a.launches), 2)
        r["hp1_physics_kernel_us_per_substep"] = round(kernel_us(tasks["morphy_stiff_unfused"], a.launches), 2)
        r["kernel_launches"] = a.launches
        out["sizes"][str(n)] = r
        for t in tasks.values():
            t.close()
        del tasks
        torch.cuda.empty_cache()
    s = json.dumps(out)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
