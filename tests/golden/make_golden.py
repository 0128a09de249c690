"""Generate golden vectors by RUNNING THE REFERENCE'S OWN CODE (this container only).

    python tests/golden/make_golden.py

Imports the reference control stack from $AERIAL_GYM_REFERENCE on CPU (see _ref_loader.py),
drives ``BaseMultirotor.step`` / ``reset_idx`` / the position-task ``compute_reward`` with
seeded inputs and stores inputs + outputs as small ``.npz`` fixtures next to this file.
The fixtures travel to the GPU box; $AERIAL_GYM_REFERENCE does not.

What is pinned: rows a1-a12, a15, a16 of SURVEY.md section 8.  What cannot be: the PhysX
integrator (a13) and Warp traversal (b9) -- not in the tree, not installable.
"""
import ast
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import _ref_loader  # noqa: E402

_ref_loader.install()

import aerial_gym.control  # noqa: E402,F401  (registers controllers)
import aerial_gym.robots  # noqa: E402,F401  (registers robots)
from aerial_gym.registry.robot_registry import robot_registry  # noqa: E402
from aerial_gym.config.env_config.empty_env import EmptyEnvCfg  # noqa: E402
from aerial_gym.utils import math as ref_math  # noqa: E402

N = 24
STEPS = 4


def rand_unit_quat(n, g):
    q = torch.randn(n, 4, generator=g)
    return q / q.norm(dim=1, keepdim=True)


def make_env_cfg(n):
    class _E(EmptyEnvCfg):
        class env(EmptyEnvCfg.env):
            num_envs = n

    return _E


# mass / inertia the oracle and product use for these robots (URDF composite inertia; see
# aerial_gym_simulator_b200/urdf.py).  The reference would take them from Isaac Gym.
ROBOT_MASS_INERTIA = {
    "base_quadrotor": (0.25, np.diag([8.45e-4, 8.45e-4, 1.69e-3])),
    "base_quad_root_link_control": (0.25, np.diag([8.45e-4, 8.45e-4, 1.69e-3])),
    "base_octarotor": (1.0, np.diag([0.02, 0.02, 0.03])),  # representative values for fixtures
    "lmf2": (1.24, np.diag([0.00252, 0.00214, 0.00436])),
}


def build_robot(robot_name, controller_name, n, num_links):
    robot, cfg = robot_registry.make_robot(robot_name, controller_name, make_env_cfg(n), "cpu")
    mass, J = ROBOT_MASS_INERTIA[robot_name]
    root = torch.zeros(n, 13)
    root[:, 6] = 1.0
    gtd = {
        "dt": 0.01,
        "gravity": torch.tensor([0.0, 0.0, -9.81]).expand(n, -1),
        "robot_state_tensor": root,
        "robot_position": root[:, 0:3],
        "robot_orientation": root[:, 3:7],
        "robot_linvel": root[:, 7:10],
        "robot_angvel": root[:, 10:13],
        "robot_force_tensor": torch.zeros(n, num_links, 3),
        "robot_torque_tensor": torch.zeros(n, num_links, 3),
        "env_bounds_min": -torch.ones(n, 3),
        "env_bounds_max": torch.ones(n, 3),
        "robot_mass": torch.full((n,), mass),
        "robot_inertia": torch.tensor(J, dtype=torch.float32).expand(n, -1, -1).clone(),
    }
    robot.init_tensors(gtd)
    return robot, cfg, gtd


def snapshot_params(robot):
    mm = robot.control_allocator.motor_model
    c = robot.controller
    out = {
        "tau_inc": mm.motor_time_constants_increasing.clone(),
        "tau_dec": mm.motor_time_constants_decreasing.clone(),
    }
    if mm.cfg.use_rps:
        out["k_thrust"] = mm.motor_thrust_constant.clone()
    if hasattr(c, "K_pos_tensor_current"):
        out["K_pos"] = c.K_pos_tensor_current.clone()
        out["K_vel"] = c.K_linvel_tensor_current.clone()
        out["K_rot"] = c.K_rot_tensor_current.clone()
        out["K_angvel"] = c.K_angvel_tensor_current.clone()
    return out


def gen_step_fixture(tag, robot_name, controller_name, num_links, num_actions, seed):
    g = torch.Generator().manual_seed(seed)
    torch.manual_seed(seed)
    robot, cfg, gtd = build_robot(robot_name, controller_name, N, num_links)
    # exercise randomised gains / motor constants where the config asks for it
    robot.controller.randomize_params(torch.arange(N))
    robot.control_allocator.reset_idx(torch.arange(N))
    rec = {}
    params = snapshot_params(robot)
    for k, v in params.items():
        rec[k] = v.numpy()
    mm = robot.control_allocator.motor_model
    root = gtd["robot_state_tensor"]
    for s in range(STEPS):
        root[:, 0:3] = torch.randn(N, 3, generator=g) * 1.5
        root[:, 3:7] = rand_unit_quat(N, g)
        if s == 0:  # near-hover attitudes too
            root[: N // 2, 3:7] = ref_math.quat_from_euler_xyz(
                torch.randn(N // 2, generator=g) * 0.2,
                torch.randn(N // 2, generator=g) * 0.2,
                torch.rand(N // 2, generator=g) * 6.28 - 3.14,
            )
        root[:, 7:10] = torch.randn(N, 3, generator=g)
        root[:, 10:13] = torch.randn(N, 3, generator=g) * 2.0
        actions = torch.rand(N, num_actions, generator=g) * 2.4 - 1.2
        if controller_name == "no_control":
            actions = torch.rand(N, num_actions, generator=g) * 2.5 - 0.25
        if s == STEPS - 1:
            actions[0] = 25.0  # clip_actions path
            actions[1] = -25.0
        rec[f"s{s}_root"] = root.clone().numpy()
        rec[f"s{s}_actions"] = actions.clone().numpy()
        rec[f"s{s}_thrust_in"] = mm.current_motor_thrust.clone().numpy()
        torch.manual_seed(seed * 100 + s)  # pins the disturbance draws (bernoulli, rand, rand)
        rec[f"s{s}_seed"] = np.array(seed * 100 + s)
        robot.step(actions.clone())
        rec[f"s{s}_thrust_out"] = mm.current_motor_thrust.clone().numpy()
        rec[f"s{s}_force"] = gtd["robot_force_tensor"].clone().numpy()
        rec[f"s{s}_torque"] = gtd["robot_torque_tensor"].clone().numpy()
        rec[f"s{s}_euler"] = gtd["robot_euler_angles"].clone().numpy()
        rec[f"s{s}_vehicle_orientation"] = gtd["robot_vehicle_orientation"].clone().numpy()
        rec[f"s{s}_vehicle_linvel"] = gtd["robot_vehicle_linvel"].clone().numpy()
        rec[f"s{s}_body_linvel"] = gtd["robot_body_linvel"].clone().numpy()
        rec[f"s{s}_body_angvel"] = gtd["robot_body_angvel"].clone().numpy()
        if hasattr(robot.controller, "wrench_command"):
            rec[f"s{s}_wrench_cmd"] = robot.controller.wrench_command.clone().numpy()
    meta = {
        "robot": robot_name,
        "controller": controller_name,
        "N": N,
        "steps": STEPS,
        "num_links": num_links,
        "application_mask": [int(x) for x in robot.application_mask.tolist()],
        "mass": ROBOT_MASS_INERTIA[robot_name][0],
        "inertia": ROBOT_MASS_INERTIA[robot_name][1].tolist(),
        "enable_disturbance": bool(cfg.disturbance.enable_disturbance),
        "prob_apply_disturbance": float(cfg.disturbance.prob_apply_disturbance),
        "max_disturbance": [float(x) for x in cfg.disturbance.max_force_and_torque_disturbance],
    }
    rec["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    np.savez_compressed(os.path.join(HERE, f"hp1_step_{tag}.npz"), **rec)
    print("wrote", tag)


def gen_reset_fixture(tag, robot_name, controller_name, num_links, seed):
    robot, cfg, gtd = build_robot(robot_name, controller_name, N, num_links)
    g = torch.Generator().manual_seed(seed)
    root = gtd["robot_state_tensor"]
    root[:, 0:3] = torch.randn(N, 3, generator=g)
    root[:, 3:7] = rand_unit_quat(N, g)
    root[:, 7:13] = torch.randn(N, 6, generator=g)
    mm = robot.control_allocator.motor_model
    rec = {"root_before": root.clone().numpy(), "thrust_before": mm.current_motor_thrust.clone().numpy()}
    for k, v in snapshot_params(robot).items():
        rec["before_" + k] = v.numpy()
    env_ids = torch.tensor([0, 3, 4, 9, 17, 23])
    torch.manual_seed(seed + 1)
    robot.reset_idx(env_ids)
    rec["seed"] = np.array(seed + 1)
    rec["env_ids"] = env_ids.numpy()
    rec["root_after"] = root.clone().numpy()
    rec["thrust_after"] = mm.current_motor_thrust.clone().numpy()
    for k, v in snapshot_params(robot).items():
        rec["after_" + k] = v.numpy()
    for k in ("euler_angles", "vehicle_orientation", "vehicle_linvel", "body_linvel", "body_angvel"):
        rec["after_" + k] = gtd["robot_" + k].clone().numpy()
    meta = {"robot": robot_name, "controller": controller_name, "N": N}
    rec["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    np.savez_compressed(os.path.join(HERE, f"hp1_reset_{tag}.npz"), **rec)
    print("wrote reset", tag)


def load_reference_reward_fn():
    """Execute the reference's compute_reward WITHOUT importing the task module (which drags
    in isaacgym / gymnasium): pull the three function defs out of the file with ``ast``."""
    path = os.path.join(
        _ref_loader.REF_ROOT, "aerial_gym/task/position_setpoint_task/position_setpoint_task.py"
    )
    src = open(path).read()
    tree = ast.parse(src)
    wanted = {"exp_func", "exp_penalty_func", "compute_reward"}
    ns = {"torch": torch, "quat_axis": ref_math.quat_axis}
    for node in tree.body:
        if isinstance(node, ast.FunctionDef) and node.name in wanted:
            node.decorator_list = []  # plain eager execution of the same arithmetic
            mod = ast.Module(body=[node], type_ignores=[])
            exec(compile(mod, path, "exec"), ns)
    return ns["compute_reward"]


def gen_reward_fixture(seed):
    g = torch.Generator().manual_seed(seed)
    n = 64
    compute_reward = load_reference_reward_fn()
    pos = torch.randn(n, 3, generator=g) * 2.0
    pos[:6] *= 6.0  # some beyond the 8 m crash radius
    q = rand_unit_quat(n, g)
    q[:20] = ref_math.quat_from_euler_xyz(
        torch.randn(20, generator=g) * 0.1, torch.randn(20, generator=g) * 0.1, torch.randn(20, generator=g)
    )
    veh_q = ref_math.vehicle_frame_quat_from_quat(rand_unit_quat(n, g))  # stale => independent of q
    body_angvel = torch.randn(n, 3, generator=g)
    linvel = torch.randn(n, 3, generator=g)
    target = torch.zeros(n, 3)
    crashes = torch.zeros(n, dtype=torch.bool)
    crashes[7] = True
    pos_err_vehicle = ref_math.quat_apply_inverse(veh_q, target - pos)
    acts = torch.zeros(n, 4)
    rew, cr = compute_reward(
        pos_err_vehicle, linvel, q, body_angvel, crashes.clone(), 1.0, acts, acts, {}
    )
    np.savez_compressed(
        os.path.join(HERE, "hp1_position_reward.npz"),
        pos=pos.numpy(), quat=q.numpy(), vehicle_orientation=veh_q.numpy(),
        body_angvel=body_angvel.numpy(), crashes_in=crashes.numpy(),
        reward=rew.numpy(), crashes_out=cr.numpy(),
    )
    print("wrote reward")


def gen_motor_csv_fixture():
    """First rows of the reference's only in-repo known-answer file (Euler, RPS space)."""
    path = os.path.join(
        _ref_loader.REF_ROOT, "aerial_gym/sim2real/motorid_utilities/sample_sim_euler_integration.csv"
    )
    rows = []
    with open(path) as f:
        for line in f:
            parts = line.strip().split(",")
            try:
                rows.append([float(p) for p in parts[:2]])
            except ValueError:
                continue
    out = {
        "source": "aerial_gym/sim2real/motorid_utilities/sample_sim_euler_integration.csv",
        "rows_t_rps": rows[:40],
        "k": 1.826312e-5, "tau": 0.04, "dt": 0.01, "rps_ref": 233.998,
    }
    json.dump(out, open(os.path.join(HERE, "motor_euler_csv.json"), "w"))
    print("wrote motor csv", len(rows))


if __name__ == "__main__":
    #            tag                    robot                        controller                   links acts seed
    CASES = [
        ("quad_attitude", "base_quadrotor", "lee_attitude_control", 9, 4, 11),
        ("quad_position", "base_quadrotor", "lee_position_control", 9, 4, 12),
        ("quad_velocity", "base_quadrotor", "lee_velocity_control", 9, 4, 13),
        ("quad_acceleration", "base_quadrotor", "lee_acceleration_control", 9, 4, 14),
        ("quad_no_control", "base_quadrotor", "no_control", 9, 4, 15),
        ("quadroot_attitude", "base_quad_root_link_control", "lee_attitude_control", 9, 4, 16),
        ("octa_velocity", "base_octarotor", "octarotor_velocity_control", 17, 4, 17),
        ("octa_fully_actuated", "base_octarotor", "rov_fully_actuated_control", 17, 7, 18),
        ("lmf2_velocity", "lmf2", "lmf2_velocity_control", 1, 4, 19),
    ]
    for c in CASES:
        gen_step_fixture(*c)
    gen_reset_fixture("quad_attitude", "base_quadrotor", "lee_attitude_control", 9, 31)
    gen_reset_fixture("octa_velocity", "base_octarotor", "octarotor_velocity_control", 17, 32)
    gen_reward_fixture(41)
    gen_motor_csv_fixture()
