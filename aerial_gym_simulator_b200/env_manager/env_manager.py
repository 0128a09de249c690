"""EnvManager -- reference surface (env_manager/env_manager.py:37-436) over Hp1Engine / RayScene /
RaySensor.  Host logic only: RNG draws (in the reference's call order), bookkeeping, the Global
Tensor Dict.  All per-env arithmetic is in the CUDA library.

Differences that are deliberate and documented (DESIGN.md):
  * no Isaac Gym: ``robot_state_tensor`` is its own contiguous [N,13] allocation (not a stride-13*A
    view of ``vec_root_tensor``); obstacles live in ``env_asset_state_tensor`` [N,K,13];
  * construction is array-native (no O(N) actor loop), except asset-file selection which keeps the
    reference's per-env ``random.choices`` / ``random.shuffle`` order;
  * contact, args['contact']:
      - "flag" (default): collision flags (a14) come from a geometric sphere-vs-mesh overlap test, not PhysX contact forces.
        Nothing stops the robot: with reset_on_collision = False it flies through obstacles and the ground.
        ``robot_contact_force_tensor`` stays 0 and ``create_ground_plane`` is not read.
      - "rigid": after every physics sub-step one velocity-level contact solve (agx_hp2_contact) stops the robot's collision
        sphere at the obstacles and, with ``create_ground_plane``, at the plane z = 0.  It fills ``robot_contact_force_tensor``,
        flags crashes by the reference's rule |F| > collision_force_threshold and adds the force to the IMU's force input.
        args['contact_friction'] is the Coulomb coefficient (default 1.0).  DESIGN.md "Contact mode" has the model.
        Obstacles are kinematic and, in the solve, at rest: dynamic_env's moving obstacles move once after the n sub-steps.
      - "rigid" with args['contact_moving_obstacles'] = True: in an env step with env_actions, every sub-step first advances the
        obstacles by one sub-step and re-poses the scene, then runs the robot's physics sub-step and the contact solve
        (agx_hp2_contact_moving), which works on the robot's velocity relative to each obstacle's velocity at the contact point.
        A moving obstacle pushes the robot, carries it by friction and flags a crash by the same force rule.  Obstacles are not
        pushed back.  The scene is re-posed every sub-step whatever args['refit_dynamic_obstacles'] says.  Steps without
        env_actions run as in plain "rigid" mode.
      - ... and args['contact_dynamic_obstacles'] = True: every obstacle asset is a free rigid body with its URDF's mass, COM and
        inertia (every asset needs fix_base_link = False).  The solve (agx_hp2_contact_dynamic) gives each impulse to the robot and,
        opposite, to the obstacle, and writes the pushed obstacles' twist and a first-order position correction to their rows.
        Every sub-step advances the obstacles, in steps without env_actions with their own damped velocity, so a knocked obstacle
        drifts; the scene is re-posed once more after the last sub-step; reset_idx zeroes the reset envs' obstacle velocities.
      - ... and args['contact_obstacle_ground'] = True (needs create_ground_plane): the free obstacles also meet the ground plane.
        Each sub-step, right after the obstacles advance, agx_obstacle_ground_contact stops every obstacle whose geometry's vertices
        are below the plane (one-body solve against the ground, the same write-back), before the scene is re-posed and the robot
        moves.
      - ... and args['contact_obstacle_obstacle'] = True: the free obstacles also collide with each other.  Every asset must be
        exactly one <box>.  Each sub-step, after the obstacle advance and the ground solve, agx_obstacle_obstacle_contact finds the
        box-box contacts of every env (separating axes, clipped faces, edge pairs) and resolves them between the two free bodies
        (the same per-contact step and write-back), before the scene is re-posed and the robot moves.
"""
from __future__ import annotations

import ctypes as C
import math
import os
import random
from collections import deque

import numpy as np
import torch

from .. import _lib
from .. import robots  # noqa: F401  (registers robots + controllers)
from .. import urdf
from ..hp1 import Hp1Engine
from ..hp2 import ContactMotion, ObstacleBoxes, ObstacleHull, ObstacleMass, RayScene, RaySensor
from ..hp2 import contact as hp2_contact
from ..hp2 import obstacle_ground_contact, obstacle_obstacle_contact
from ..registry._core import env_config_registry, robot_registry, sim_config_registry


def _lerp(lo, hi, u):  # utils/math.py:51-54 torch_rand_float_tensor arithmetic
    return (hi - lo) * u + lo


def _quat_from_euler(e):  # utils/math.py:155-172
    roll, pitch, yaw = e[..., 0], e[..., 1], e[..., 2]
    cy, sy = torch.cos(yaw * 0.5), torch.sin(yaw * 0.5)
    cr, sr = torch.cos(roll * 0.5), torch.sin(roll * 0.5)
    cp, sp = torch.cos(pitch * 0.5), torch.sin(pitch * 0.5)
    return torch.stack([cy * sr * cp - sy * cr * sp, cy * cr * sp + sy * sr * cp, sy * cr * cp - cy * sr * sp,
                        cy * cr * cp + sy * sr * sp], dim=-1)


def _quat_mul(a, b):  # xyzw Hamilton product
    ax, ay, az, aw = a.unbind(-1)
    bx, by, bz, bw = b.unbind(-1)
    return torch.stack([aw * bx + bw * ax + ay * bz - az * by, aw * by + bw * ay + az * bx - ax * bz,
                        aw * bz + bw * az + ax * by - ay * bx, aw * bw - ax * bx - ay * by - az * bz], dim=-1)


def _matrix_to_quat(R):
    """xyzw quaternion of a rotation matrix (Shepperd's method, float64)"""
    t = np.trace(R)
    if t > 0:
        s = 2.0 * np.sqrt(1.0 + t)
        return np.array([(R[2, 1] - R[1, 2]) / s, (R[0, 2] - R[2, 0]) / s, (R[1, 0] - R[0, 1]) / s, 0.25 * s])
    i = int(np.argmax(np.diag(R)))
    j, k = (i + 1) % 3, (i + 2) % 3
    s = 2.0 * np.sqrt(1.0 + R[i, i] - R[j, j] - R[k, k])
    v = np.zeros(4)
    v[i], v[j], v[k], v[3] = 0.25 * s, (R[j, i] + R[i, j]) / s, (R[k, i] + R[i, k]) / s, (R[k, j] - R[j, k]) / s
    return v


def _obstacle_mass_row(model, path):
    """the AgxObstacleMass row of a free obstacle asset: the composite mass properties of its URDF inertials (the robot's come from
    the same function).  No density is assumed: an asset without mass is an error."""
    m, com, J = model.composite_inertia()
    if not m > 0:
        raise ValueError(f"{path}: a free obstacle asset needs URDF inertials with a total mass > 0")
    if not np.linalg.matrix_rank(J) == 3:
        raise ValueError(f"{path}: the composite inertia of a free obstacle asset must be invertible")
    return ObstacleMass.row(m, com, J)


def _hull_vertices(parts):
    """the distinct vertices of an asset's scene parts (urdf.visual_parts, asset frame), in order of first appearance"""
    v = np.concatenate([t.reshape(-1, 3) for _, _, t, _ in parts]) if parts else np.zeros((0, 3), np.float32)
    _, first = np.unique(v, axis=0, return_index=True)
    return v[np.sort(first)]


def _obstacle_box_row(parts, path):
    """the ObstacleBoxes row of a free obstacle asset whose scene parts (urdf.visual_parts) are exactly one <box>"""
    if len(parts) != 1 or parts[0][3] is None or parts[0][3][15] != 2.0:
        raise ValueError(f"{path}: args['contact_obstacle_obstacle'] needs every obstacle asset to be exactly one <box>")
    return ObstacleBoxes.row(parts[0][3])


def _quat_rotate_inverse(q, v):
    qw, qv = q[:, 3:4], q[:, 0:3]
    return v * (2.0 * qw * qw - 1.0) - torch.cross(qv, v, dim=-1) * qw * 2.0 + qv * (qv * v).sum(-1, keepdim=True) * 2.0


class _RobotManagerView:
    """robots/robot_manager.py: RobotManagerIGE as callers see it (the arithmetic it hosts in the reference runs in the HP1 kernel)"""

    def __init__(self, env):
        self._env, self.robot, self.cfg = env, env.robot, env.robot_cfg
        self.num_envs, self.device = env.num_envs, env.device
        self.robot_mass, self.robot_inertia = env.robot.robot_mass, env.robot.robot_inertia  # :45-46, scalars / 3x3 of the URDF
        self.dof_control_mode = "none"

    robot_masses = property(lambda self: self._env.global_tensor_dict["robot_mass"])      # :47  [N]
    robot_inertias = property(lambda self: self._env.global_tensor_dict["robot_inertia"])  # :48  [N,3,3]
    imu_sensor = property(lambda self: self._env.imu)
    warp_sensor = lidar_sensor = property(lambda self: self._env.sensor)
    camera_sensor = property(lambda self: None)  # Isaac Gym's rasterised cameras do not exist here


class _SimView:
    """env_manager/IGE_env_manager.py: the counts callers read off IsaacGymEnv"""

    def __init__(self, env):
        self._env, self.sim_config, self.num_envs = env, env.sim_config, env.num_envs
        self.sim_has_dof, self.dof_control_mode, self.viewer, self.has_viewer = env.articulated, "none", None, False

    num_assets_per_env = property(lambda self: self._env.num_obs_in_env + 1)  # :269-276, the robot is an actor too
    num_rigid_bodies_robot = property(lambda self: self._env.robot.num_bodies)
    global_tensor_dict = property(lambda self: self._env.global_tensor_dict)


class EnvManager:
    def __init__(self, sim_name, env_name, robot_name, controller_name, device, args=None, num_envs=None,
                 use_warp=None, headless=None):
        self.robot_name, self.controller_name = robot_name, controller_name
        self.sim_config = sim_config_registry.make_sim(sim_name)
        self.cfg = env_config_registry.make_env(env_name)
        self.device = torch.device(device)
        if num_envs is not None:
            self.cfg.env.num_envs = num_envs
        if use_warp is not None:
            self.cfg.env.use_warp = use_warp
        if headless is not None:
            self.sim_config.viewer.headless = headless
        self.num_envs = self.cfg.env.num_envs
        self.use_warp = self.cfg.env.use_warp
        self.env_args = dict(args or {})
        # "device": in-kernel Philox resets, no host round trip (default).
        # "torch" : uniforms drawn with torch.rand in the reference's call order, host sync per step
        #           exactly where the reference has one (env_manager.py:364-375).
        self.reset_rng = self.env_args.get("reset_rng", "device")
        if self.reset_rng not in ("device", "torch"):
            raise ValueError("args['reset_rng'] must be 'device' or 'torch'")
        self.contact_mode = self.env_args.get("contact", "flag")
        if self.contact_mode not in ("flag", "rigid"):
            raise ValueError("args['contact'] must be 'flag' or 'rigid'")
        mu = self.env_args.get("contact_friction", 1.0)
        if isinstance(mu, bool) or not isinstance(mu, (int, float)) or not math.isfinite(mu) or mu < 0:
            raise ValueError("args['contact_friction'] must be a finite number >= 0")
        self.contact_friction = float(mu)
        moving = self.env_args.get("contact_moving_obstacles", False)
        if not isinstance(moving, bool):
            raise ValueError("args['contact_moving_obstacles'] must be a bool")
        if moving and self.contact_mode != "rigid":
            raise ValueError("args['contact_moving_obstacles'] needs args['contact'] = 'rigid'")
        self.contact_moving_obstacles = moving
        dynamic = self.env_args.get("contact_dynamic_obstacles", False)
        if not isinstance(dynamic, bool):
            raise ValueError("args['contact_dynamic_obstacles'] must be a bool")
        if dynamic and not moving:
            raise ValueError("args['contact_dynamic_obstacles'] needs args['contact_moving_obstacles'] = True")
        self.contact_dynamic_obstacles = dynamic
        ground = self.env_args.get("contact_obstacle_ground", False)
        if not isinstance(ground, bool):
            raise ValueError("args['contact_obstacle_ground'] must be a bool")
        if ground and not dynamic:
            raise ValueError("args['contact_obstacle_ground'] needs args['contact_dynamic_obstacles'] = True")
        if ground and not bool(getattr(self.cfg.env, "create_ground_plane", False)):
            raise ValueError("args['contact_obstacle_ground'] needs an env with create_ground_plane")
        self.contact_obstacle_ground = ground
        pairs = self.env_args.get("contact_obstacle_obstacle", False)
        if not isinstance(pairs, bool):
            raise ValueError("args['contact_obstacle_obstacle'] must be a bool")
        if pairs and not dynamic:
            raise ValueError("args['contact_obstacle_obstacle'] needs args['contact_dynamic_obstacles'] = True")
        self.contact_obstacle_obstacle = pairs
        self.global_tensor_dict = {}
        self.step_counter = 0
        self._graphs, self._dist_ctr_dev = {}, None
        self._populate()
        # "graph" (default where it applies): the per-sub-step launches of an env step with obstacles / disturbances replay as one CUDA
        # graph; "launch": one C-ABI call per kernel, as in round 1.  The torch-order RNG mode draws with torch inside the loop: launches.
        want = self.env_args.get("step_mode", "graph")
        if want not in ("graph", "launch"):
            raise ValueError("args['step_mode'] must be 'graph' or 'launch'")
        self.step_mode = want if (self.reset_rng == "device" and self.device.type == "cuda") else "launch"
        self.sim_steps = self.engine.sim_steps  # int32 [N] (env_manager.py:78-80)
        # the reference's object graph, as far as its examples / tasks / trainers walk it: env.robot_manager.robot.{cfg, controller,
        # controller_config}, env.IGE_env.num_assets_per_env (robot included, IGE_env_manager.py:269-276)
        self.robot_manager = _RobotManagerView(self)
        self.IGE_env = _SimView(self)

    # ------------------------------------------------------------------------------------------
    # construction (populate_env + prepare_sim, env_manager.py:127-271)
    # ------------------------------------------------------------------------------------------
    def _populate(self):
        N, dev = self.num_envs, self.device
        self.robot, self.robot_cfg = robot_registry.make_robot(self.robot_name, self.controller_name, self.cfg, dev)
        self.num_robot_actions = self.robot.num_actions
        spec = self.robot.make_spec(self.sim_config, self.cfg)
        self.spec = spec
        self.articulated = bool(getattr(self.robot, "articulated", False))
        articulation = None
        imu_on = bool(getattr(self.robot_cfg.sensor_config, "enable_imu", False))
        imu_link = getattr(self.robot_cfg.sensor_config.imu_config, "parent_link", None) if imu_on else None
        # an IMU on a link (imu_config.parent_link): (link name, body, R_l = the link's frame in the body's frame)
        self._imu_link = (imu_link, *self._resolve_link(imu_link)[:2]) if imu_link is not None else None
        if self.articulated:
            if self.contact_mode == "rigid":
                raise ValueError("args['contact'] = 'rigid' is not available for an articulated robot: the contact solve gives its impulse "
                                 "to the base alone, which is wrong for a tree of bodies")
            if imu_on and imu_link is None:
                raise ValueError("the IMU of an articulated robot reads the force on one body, the joint reaction forces included: "
                                 "name the link with imu_config.parent_link")
            if imu_on and not self.robot.bodies.mass[self._imu_link[1]] > 0:
                raise ValueError(f"imu_config.parent_link '{imu_link}' belongs to a body without mass: the IMU divides its force by the "
                                 "body's mass")
            if bool(self.env_args.get("host_io", False)):
                raise NotImplementedError("args['host_io'] is a feature of the fused task step, which articulated robots do not have")
            articulation = self.robot.make_articulation()
        extra = {"articulation": articulation} if articulation is not None else {}
        if articulation is not None and imu_on:
            extra["imu_body"] = self._imu_link[1]  # the step also writes that body's force input (Hp1Engine.imu_input)
        # joint force sensing (Isaac Gym's enable_dof_force_sensors): the step also writes every joint's wrench and DOF force
        if getattr(getattr(self.robot_cfg, "joint_config", None), "enable_dof_force_sensors", False):
            extra["joint_force"] = True
        self.engine = Hp1Engine(
            spec, N, dev, physics_steps=1, seed=int(self.env_args.get("seed", 0)),
            env_id_offset=int(self.env_args.get("env_id_offset", 0)), device_rng_reset=(self.reset_rng == "device"),
            strict_stale_obs=bool(self.env_args.get("strict_stale_obs", True)), materialize_derived=True,
            per_env_params=self.env_args.get("per_env_params", "auto"), host_io=bool(self.env_args.get("host_io", False)),
            debug_wrench=imu_on and not self.articulated,  # a rigid robot's IMU reads the net body force
            **extra)
        eng, gtd = self.engine, self.global_tensor_dict
        if articulation is not None:
            # joint state (position, velocity) and the drive targets; the targets belong to the user: the env never writes them
            gtd["dof_state_tensor"] = eng.dof_state
            gtd["dof_position_setpoint_tensor"] = eng.dof_position_setpoint
            gtd["dof_velocity_setpoint_tensor"] = eng.dof_velocity_setpoint
            if getattr(eng, "dof_actuation_force", None) is not None:  # the commanded torques of the effort DOFs, the user's too
                gtd["dof_actuation_force_tensor"] = eng.dof_actuation_force
            if getattr(eng, "dof_force", None) is not None:  # written by every step, rows of the wrench in robot_body_names order
                gtd["dof_force_tensor"] = eng.dof_force
                gtd["robot_joint_wrench_tensor"] = eng.joint_wrench
            T = lambda v: torch.tensor(np.asarray(v, np.float32), device=dev)
            self._dof_rng = tuple(T(r) for r in (*articulation.init_dof_pos_range, *articulation.init_dof_vel_range))
        # every body's pose and velocity [N,B,13] (rows like robot_state_tensor's, body 0 = the root link), refreshed once per env step
        self._body_state = getattr(eng, "body_state", None) if articulation is not None else None
        if self._body_state is not None:
            gtd["robot_body_state_tensor"] = self._body_state
            gtd["robot_body_names"] = list(articulation.bodies.links)
        self.robot.controller.bind_engine(eng)  # controller.K_*_tensor_current / set_controller_gains act on the engine's gains
        gtd["crashes"], gtd["truncations"] = eng.terminations, eng.truncations
        self.collision_tensor, self.truncation_tensor = eng.terminations, eng.truncations
        self.num_env_actions = self.cfg.env.num_env_actions
        gtd["num_env_actions"], gtd["env_actions"], gtd["prev_env_actions"] = self.num_env_actions, None, None
        # robot tensors (IGE_env_manager.py:301-311, base_multirotor.py:85-91, robot_manager.py:112-126)
        rs = eng.root_state
        gtd["robot_state_tensor"] = rs
        gtd["robot_position"], gtd["robot_orientation"] = rs[:, 0:3], rs[:, 3:7]
        gtd["robot_linvel"], gtd["robot_angvel"] = rs[:, 7:10], rs[:, 10:13]
        gtd["robot_euler_angles"], gtd["robot_vehicle_orientation"] = eng.euler, eng.vehicle_orientation
        gtd["robot_vehicle_linvel"], gtd["robot_body_linvel"], gtd["robot_body_angvel"] = (
            eng.vehicle_linvel, eng.body_linvel, eng.body_angvel)
        gtd["robot_actions"] = torch.zeros(N, self.num_robot_actions, device=dev)
        gtd["robot_prev_actions"] = torch.zeros_like(gtd["robot_actions"])
        gtd["num_robot_actions"] = self.num_robot_actions
        gtd["robot_mass"] = torch.full((N,), float(self.robot.robot_mass), device=dev)
        gtd["robot_inertia"] = torch.tensor(self.robot.robot_inertia, dtype=torch.float32, device=dev).expand(N, -1, -1)
        B = self.robot.num_bodies
        gtd["robot_force_tensor"] = torch.zeros(N, B, 3, device=dev)   # not materialised by the fused step
        gtd["robot_torque_tensor"] = torch.zeros(N, B, 3, device=dev)
        gtd["robot_contact_force_tensor"] = torch.zeros(N, 3, device=dev)
        gtd["env_bounds_min"], gtd["env_bounds_max"] = eng.bounds_min, eng.bounds_max
        gtd["gravity"] = torch.tensor(self.sim_config.sim.gravity, device=dev).expand(N, -1)
        gtd["dt"] = self.sim_config.sim.dt
        gtd["dof_control_mode"] = "none"
        self._bounds_rng = tuple(torch.tensor(v, dtype=torch.float32, device=dev) for v in (
            self.cfg.env.lower_bound_min, self.cfg.env.lower_bound_max, self.cfg.env.upper_bound_min, self.cfg.env.upper_bound_max))
        # IsaacGymEnv.__init__ draws the initial bounds (IGE_env_manager.py:59-64)
        eng.bounds_min.copy_(_lerp(self._bounds_rng[0], self._bounds_rng[1], torch.rand(N, 3, device=dev)))
        eng.bounds_max.copy_(_lerp(self._bounds_rng[2], self._bounds_rng[3], torch.rand(N, 3, device=dev)))
        self._build_obstacles()
        self._build_sensors()
        self._update_body_state()  # the rows of the creation pose, until the first reset
        if eng.host_io and (self.scene is not None or self.reset_rng != "device" or self.contact_mode == "rigid"):
            raise NotImplementedError("args['host_io'] needs an obstacle-free env, reset_rng='device' and contact='flag': the flags "
                                      "live in host memory and are written only by the fused task step")
        self.contact_params = None
        if self.contact_mode == "rigid":
            px, c = self.sim_config.sim.physx, eng.cfg
            p = self.contact_params = _lib.AgxContactParams()
            p.radius, p.contact_offset, p.rest_offset = float(self.robot.collision_radius), float(px.contact_offset), float(px.rest_offset)
            p.dt, p.mass = float(self.sim_config.sim.dt), float(c.mass)
            p.inertia_inv[:], p.com[:] = list(c.inertia_inv), list(c.com)
            p.friction, p.max_depenetration_velocity = self.contact_friction, float(px.max_depenetration_velocity)
            p.force_threshold = float(self.cfg.env.collision_force_threshold)
            p.iterations, p.ground_plane = int(px.num_position_iterations), int(bool(getattr(self.cfg.env, "create_ground_plane", False)))
        # the moving-obstacle solve reads the asset rows through the object -> asset map (int32, range-checked once here)
        self._contact_motion = None
        if self.contact_moving_obstacles and self.scene is not None:
            self._contact_motion = ContactMotion(self.global_tensor_dict["env_asset_state_tensor"], self._obj_asset)
        # the dynamic-obstacle solve: every asset a free body with its URDF's mass properties (table built in _build_obstacles)
        self._obstacle_mass = None
        if self._contact_motion is not None and self.contact_dynamic_obstacles:
            self._obstacle_mass = ObstacleMass(self._asset_mass.to(dev))
        # the obstacle-ground solve: every asset's vertices (table built in _build_obstacles)
        self._obstacle_hull = None
        if self._obstacle_mass is not None and self.contact_obstacle_ground:
            self._obstacle_hull = ObstacleHull.from_files(self._hull_files, self._asset_file, dev)
        # the obstacle-obstacle solve: every asset's box (table built in _build_obstacles)
        self._obstacle_boxes = None
        if self._obstacle_mass is not None and self.contact_obstacle_obstacle:
            self._obstacle_boxes = ObstacleBoxes(torch.from_numpy(np.stack(self._box_rows)).to(dev),
                                                 torch.from_numpy(self._asset_box).to(dev))

    # ---- obstacles: AssetLoader.select_assets_for_sim + WarpEnv (asset_loader.py:148-194, warp_env_manager.py)
    def _select_assets(self):
        ec = self.cfg.env_config
        ordered, keep = deque(), 0
        for asset_type, params in ec.asset_type_to_dict_map.items():
            if asset_type in ec.include_asset_type and ec.include_asset_type[asset_type] is False:
                continue
            n = params.num_assets
            if n <= 0:
                continue
            if params.file is None:
                files = sorted(f for f in os.listdir(params.asset_folder) if f.endswith(".urdf"))
                chosen = random.choices(files, k=n)
            else:
                chosen = [params.file] * n
            for f in chosen:
                item = (params, os.path.join(params.asset_folder, f))
                if params.keep_in_env:
                    ordered.appendleft(item)
                    keep += 1
                else:
                    ordered.append(item)
        ordered = list(ordered)
        tail = ordered[keep:]
        random.shuffle(tail)
        ordered[keep:] = tail
        return ordered, keep

    def _build_obstacles(self):
        N, dev, gtd = self.num_envs, self.device, self.global_tensor_dict
        self.scene = None
        per_env, self.keep_in_env = [], 0
        if self.cfg.env_config.asset_type_to_dict_map:
            for _ in range(N):
                sel, keep = self._select_assets()
                per_env.append(sel)
                self.keep_in_env = keep
        A = len(per_env[0]) if per_env else 0
        if any(len(s) != A for s in per_env):
            raise ValueError("All environments should have the same number of assets")
        # dynamic obstacles (agx_obstacle_step): one pair of damping coefficients for the whole scene -- every shipped asset
        # class has 0.1 / 0.1 (config/asset_config/*_config.py: asset_state_params)
        p0 = per_env[0][0][0] if A else None
        self._asset_damping = (float(getattr(p0, "linear_damping", 0.0)), float(getattr(p0, "angular_damping", 0.0)))
        self.num_obs_in_env = A
        gtd["num_obstacles_in_env"] = A
        gtd["env_asset_state_tensor"] = torch.zeros(N, A, 13, device=dev)
        if A:
            gtd["env_asset_state_tensor"][..., 6] = 1.0
        gtd["asset_min_state_ratio"] = torch.zeros(N, A, 13, device=dev)
        gtd["asset_max_state_ratio"] = torch.zeros(N, A, 13, device=dev)
        if not A:
            return
        ast = gtd["env_asset_state_tensor"]
        gtd["obstacle_position"], gtd["obstacle_orientation"] = ast[..., 0:3], ast[..., 3:7]
        gtd["obstacle_linvel"], gtd["obstacle_angvel"] = ast[..., 7:10], ast[..., 10:13]
        lo = np.zeros((N, A, 13), np.float32)
        hi = np.zeros((N, A, 13), np.float32)
        # templates: every visual of every distinct URDF; an asset with b parts = b objects sharing its pose (a box is one part, a
        # tessellated cylinder eleven, a <mesh> / <sphere> one mesh object: urdf.visual_parts).  Mesh parts are numbered after
        # every cluster template (RayScene's mesh_templates).
        templates, tmpl_obbs, boxes_of, tmpl_link = [], [], {}, []
        meshes, mesh_link = [], []
        # dynamic obstacles: one mass-table row per distinct URDF (inverse mass, COM, inverse inertia: AgxObstacleMass)
        dynamic = self.contact_dynamic_obstacles
        mass_of, asset_mass = {}, (np.zeros((N, A, 13), np.float32) if dynamic else None)
        # obstacle-ground contact: the vertices of each distinct URDF's scene parts, and each asset's file
        ground = self.contact_obstacle_ground
        file_of, hull_files, asset_file = {}, [], (np.zeros((N, A), np.int32) if ground else None)
        # obstacle-obstacle contact: the box of each distinct URDF, and each asset's box
        pairs = self.contact_obstacle_obstacle
        box_of, box_rows, asset_box = {}, [], (np.zeros((N, A), np.int32) if pairs else None)
        for e in range(N):
            for a, (params, path) in enumerate(per_env[e]):
                lo[e, a], hi[e, a] = params.min_state_ratio, params.max_state_ratio
                if dynamic and getattr(params, "fix_base_link", True):
                    raise ValueError(f"args['contact_dynamic_obstacles'] needs every obstacle asset to have fix_base_link = False "
                                     f"({getattr(params, '__name__', type(params).__name__)} has a fixed base link)")
                if path not in boxes_of:
                    model = urdf.parse_urdf(path)
                    if dynamic:
                        mass_of[path] = _obstacle_mass_row(model, path)
                    ids = []
                    parts = urdf.visual_parts(model, params.use_collision_mesh_instead_of_visual)
                    if ground:
                        file_of[path] = len(hull_files)
                        hull_files.append(_hull_vertices(parts))
                    if pairs:
                        box_of[path] = len(box_rows)
                        box_rows.append(_obstacle_box_row(parts, path))
                    for _, link_index, tris, obb in parts:
                        if obb is None:
                            ids.append(-1 - len(meshes))
                            meshes.append(tris)
                            mesh_link.append(link_index)
                            continue
                        ids.append(len(templates))
                        templates.append(tris)
                        tmpl_obbs.append(obb)
                        tmpl_link.append(link_index)
                    boxes_of[path] = ids
                if dynamic:
                    asset_mass[e, a] = mass_of[path]
                if ground:
                    asset_file[e, a] = file_of[path]
                if pairs:
                    asset_box[e, a] = box_of[path]
        if dynamic:
            self._asset_mass = torch.from_numpy(asset_mass)
        if ground:
            self._hull_files, self._asset_file = hull_files, asset_file
        if pairs:
            self._box_rows, self._asset_box = box_rows, asset_box
        gtd["asset_min_state_ratio"].copy_(torch.from_numpy(lo))
        gtd["asset_max_state_ratio"].copy_(torch.from_numpy(hi))
        if not self.use_warp:
            return
        T = len(templates)
        boxes_of = {p: [t if t >= 0 else T - 1 - t for t in ids] for p, ids in boxes_of.items()}
        tmpl_link += mesh_link
        tmpl_obbs += [np.zeros(16, np.float32)] * len(meshes)
        templates_all = templates + meshes
        nb = [sum(len(boxes_of[p]) for _, p in per_env[e]) for e in range(N)]
        K = max(nb)
        if K == 0:
            return
        obj_t = np.zeros((N, K), np.int32)
        obj_c = np.zeros((N, K), np.int32)
        obj_asset = np.zeros((N, K), np.int64)
        seg_base, seg_mask = [0] * len(templates_all), [0] * len(templates_all)
        seg_ctr = 100  # env_manager.py:147; global across envs like the reference
        for e in range(N):
            k = 0
            for a, (params, path) in enumerate(per_env[e]):
                per_link = bool(getattr(params, "per_link_semantic", False))
                for t in boxes_of[path]:
                    obj_t[e, k], obj_asset[e, k] = t, a
                    if per_link:  # one id per link: link counter + the env's running counter (warp_asset.py:44-70, e.g. the trees)
                        seg_base[t], seg_mask[t], obj_c[e, k] = tmpl_link[t], 1, seg_ctr
                    elif params.semantic_id < 0:  # per-instance id = counter (warp_asset.py:100-104, warp_env_manager.py:76-80)
                        seg_base[t], seg_mask[t], obj_c[e, k] = 0, 1, seg_ctr
                    else:
                        seg_base[t], seg_mask[t], obj_c[e, k] = params.semantic_id, 0, 0
                    k += 1
                # the running counter advances by the number of distinct variable ids the asset used (warp_env_manager.py:90-95)
                seg_ctr += (max(tmpl_link[t] for t in boxes_of[path]) + 1) if (per_link and boxes_of[path]) else 1
            while k < K:  # pad ragged envs with a repeat of the last object (same pose, same id)
                obj_t[e, k], obj_c[e, k], obj_asset[e, k] = obj_t[e, k - 1], obj_c[e, k - 1], obj_asset[e, k - 1]
                k += 1
        # object poses: one row per object, gathered from the asset rows after every asset reset
        self._obj_asset = torch.from_numpy(obj_asset).to(dev)
        self._obj_pose = torch.zeros(N, K, 7, device=dev)
        self.scene = RayScene(templates, seg_base, seg_mask, obj_t, obj_c, self._obj_pose, dev,
                              bounds_min=self.engine.bounds_min, bounds_max=self.engine.bounds_max,
                              tmpl_obb=np.stack(tmpl_obbs), **({"mesh_templates": meshes} if meshes else {}))  # keyword only when used
        # Until the first reset_idx every actor sits where it was created: at the env origin, identity orientation
        # (IGE_env_manager.py: create_actor with the default start pose), the robot among them.  Tasks whose reset() does not reset the
        # sim (NavigationTask.reset, navigation_task.py:162-175) therefore begin in contact: the first step flags a crash and the
        # first real episode starts with the reset that follows.  Build the scene for that configuration.
        self._obj_pose[..., 6] = 1.0
        self.scene.update()

    def _build_sensors(self):
        gtd, N, dev = self.global_tensor_dict, self.num_envs, self.device
        sc = self.robot_cfg.sensor_config
        self.sensor, self.sensor_cfg, self._sensor_link = None, None, None
        self.imu = None
        if getattr(sc, "enable_imu", False):  # robot_manager.py:91-96, 246-262
            from ..sensors import IMUSensor
            # PhysX's force sensor reports the TOTAL force on the link, gravity included (base_imu_config.py:48), in the link
            # frame: here = applied base-frame force of the last physics step + m R(q)^T g  (refreshed in render_sensors)
            gtd["force_sensor_tensor"] = torch.zeros(N, 6, device=dev)
            self.imu = IMUSensor(sc.imu_config, N, dev)
            self.imu.init_tensors(gtd)
            if self._imu_link is not None:
                # an IMU on a link: sensor_quats stays relative to the link, the kernel reads q_l (x) sensor_quats
                _, b, R_l = self._imu_link
                self.imu.set_link(torch.tensor(_matrix_to_quat(np.asarray(R_l, np.float64)), dtype=torch.float32))
                if self.articulated:
                    # ... and body b's force input (Hp1Engine.imu_input), mass, orientation row and angular velocity
                    self._imu_mass = torch.full((N,), float(self.robot.bodies.mass[b]), device=dev)
                    self._imu_angvel = torch.zeros(N, 3, device=dev)
                    self.imu.robot_masses, self.imu.robot_state = self._imu_mass, self._body_state[:, b, :]
                    self.imu.robot_body_angvel = self._imu_angvel
        if not self.use_warp:
            return
        if sc.enable_camera and sc.enable_lidar:
            raise ValueError("Both camera and lidar are enabled: they share depth_range_pixels (robot_manager.py:69-89).")
        cfg = sc.camera_config if sc.enable_camera else (sc.lidar_config if sc.enable_lidar else None)
        if cfg is None:
            return
        if self.scene is None:
            return  # "Warp camera is enabled but there is nothing in the environment" (robot_manager.py:189-192)
        S, H, W = cfg.num_sensors, cfg.height, cfg.width
        pc = bool(cfg.return_pointcloud)
        gtd["depth_range_pixels"] = torch.zeros((N, S, H, W, 3) if pc else (N, S, H, W), device=dev)
        seg = None
        if cfg.segmentation_camera:
            seg = gtd["segmentation_pixels"] = torch.zeros(N, S, H, W, dtype=torch.int32, device=dev)
        self.sensor_cfg = cfg
        T = lambda v: torch.tensor(v, dtype=torch.float32, device=dev)
        self._mount_rng = (T(cfg.min_translation), T(cfg.max_translation),
                           torch.deg2rad(T(cfg.min_euler_rotation_deg)), torch.deg2rad(T(cfg.max_euler_rotation_deg)))
        self.sensor_mount = torch.zeros(N, S, 7, device=dev)
        mean_e = (self._mount_rng[2] + self._mount_rng[3]) / 2.0  # warp_sensor.py:118-123
        self.sensor_mount[..., 3:7] = _quat_from_euler(mean_e.expand(N, S, 3))
        # a sensor on a link (cfg.parent_link): pose = body pose o T_l o mount o frame rotation.  The cast reads the link's body row
        # of robot_body_state_tensor (robot_state_tensor on a robot without joints) and a mount with T_l folded in; sensor_mount
        # stays relative to the link
        pose, mount = self.engine.root_state, self.sensor_mount
        link = getattr(cfg, "parent_link", None)
        if link is not None:
            b, R_l, p_l = self._resolve_link(link)
            if self._body_state is not None:
                pose = self._body_state[:, b, :]
            elif b != 0:
                raise ValueError(f"sensor parent_link '{link}' moves with a joint, and the engine publishes no per-body state")
            T = lambda v: torch.tensor(np.asarray(v, np.float32), device=dev)
            self._sensor_link = (T(R_l), T(p_l), T(_matrix_to_quat(np.asarray(R_l, np.float64))))
            mount = self.sensor_mount_body = torch.zeros(N, S, 7, device=dev)
            self._fold_link_into_mount()
        self.sensor = RaySensor(cfg, self.scene, pose, gtd["depth_range_pixels"], seg, mount)
        self.sensor.mount = mount  # keep the live tensor (RaySensor made it contiguous already)
        self.sensor.c.mount = mount.data_ptr()
        # sensor noise (WarpSensor.apply_noise, warp_sensor.py:227-250): "device" = one in-place pass with a counter-based
        # device RNG (agx_hp2_noise_limits; default next to the in-kernel Philox resets), "torch" = the reference's torch calls
        # in the reference's order (default when reset_rng == "torch", i.e. when every random number comes from torch)
        self.sensor_noise_rng = self.env_args.get("sensor_noise_rng", "device" if self.reset_rng == "device" else "torch")
        if self.sensor_noise_rng not in ("device", "torch"):
            raise ValueError("args['sensor_noise_rng'] must be 'device' or 'torch'")
        self._device_noise = None
        if self.sensor.noise_enabled and self.sensor_noise_rng == "device":
            from ..sensors.noise import DeviceSensorNoise
            px = gtd["depth_range_pixels"]
            per_env = px[0].numel() // (3 if pc else 1)
            self._device_noise = DeviceSensorNoise(cfg, px, seed=int(self.env_args.get("seed", 0)) ^ 0x5E4503_4E015E,
                                                   first_pixel=int(self.env_args.get("env_id_offset", 0)) * per_env)

    def _resolve_link(self, name):
        """(body, R_l, p_l): the body a URDF link belongs to and the link's frame in that body's frame (on a robot without joints:
        body 0 and the link's fixed transform from the root link)"""
        model = self.robot.urdf_model
        if name not in model.links:
            raise ValueError(f"sensor parent_link '{name}' is not a link of robot '{self.robot_name}'; its links are {sorted(model.links)}")
        if self.articulated:
            R, p = self.robot.bodies.link_in_body[name]
            return self.robot.bodies.link_body[name], R, p
        R, p = model.link_transforms()[name]
        return 0, R, p

    def _fold_link_into_mount(self):
        """sensor_mount_body = T_l o sensor_mount (position p_l + R_l m_p, orientation q_l (x) m_q), after every mount draw"""
        R, p, q = self._sensor_link
        m = self.sensor_mount
        self.sensor_mount_body[..., 0:3] = p + (R * m[..., None, 0:3]).sum(-1)
        self.sensor_mount_body[..., 3:7] = _quat_mul(q.expand_as(m[..., 3:7]), m[..., 3:7])

    # ------------------------------------------------------------------------------------------
    # reset (env_manager.py:273-301)
    # ------------------------------------------------------------------------------------------
    def _reset_assets(self, env_ids, num_obstacles):
        """AssetManager.reset_idx (asset_manager.py:51-71): full-size draw, gather, park the rest."""
        gtd = self.global_tensor_dict
        ast = gtd["env_asset_state_tensor"]
        n_keep = max(num_obstacles, self._num_keep)
        lo, hi = gtd["asset_min_state_ratio"], gtd["asset_max_state_ratio"]
        r = _lerp(lo, hi, torch.rand_like(hi))
        bmin = self.engine.bounds_min.unsqueeze(1)
        bmax = self.engine.bounds_max.unsqueeze(1)
        pos = bmin + (bmax - bmin) * r[..., 0:3]
        ast[env_ids, :, 0:3] = pos[env_ids]
        ast[env_ids, :, 3:7] = _quat_from_euler(r[env_ids][..., 3:6])
        ast[env_ids, n_keep:, 0:3] = -1000.0

    def reset_idx(self, env_ids=None):
        eng, gtd, dev, N = self.engine, self.global_tensor_dict, self.device, self.num_envs
        if env_ids is None:
            env_ids = torch.arange(N, device=dev)
        env_ids = env_ids.to(dev)
        mask = torch.zeros(N, dtype=torch.bool, device=dev)
        mask[env_ids] = True
        A = gtd["num_obstacles_in_env"]
        # robots whose reset leaves the motor model alone (BaseROV, robots/base_rov.py:188-201): put it back after the engine's reset
        motor_names = ("motor_thrust", "tau_inc", "tau_dec", "k_thrust")
        saved_motors = None
        if getattr(self.robot, "keeps_motor_state_on_reset", False) and getattr(self, "_motors_initialised", False):
            saved_motors = {k: getattr(eng, k).clone() for k in motor_names if getattr(eng, k, None) is not None}
        if self.reset_rng == "device":
            # Philox reset of bounds + robot + motor/controller params in one launch; the asset
            # sampling below only needs the new bounds (reference order: bounds -> assets -> robot,
            # and the robot sampling does not depend on the assets)
            eng.reset(mask, None)
            if A > 0:
                self._sample_assets_and_update_scene(env_ids, mask, A)
        else:
            M = self.spec.num_motors
            r = lambda *s: torch.rand(*s, device=dev)
            # IsaacGymEnv.reset_idx: two full-size draws (IGE_env_manager.py:513-519)
            draws = {"bounds_lo": r(N, 3), "bounds_hi": r(N, 3)}
            if A > 0:
                lo0, lo1, hi0, hi1 = self._bounds_rng
                eng.bounds_min[env_ids] = _lerp(lo0, lo1, draws["bounds_lo"])[env_ids]
                eng.bounds_max[env_ids] = _lerp(hi0, hi1, draws["bounds_hi"])[env_ids]
                self._sample_assets_and_update_scene(env_ids, mask, A)
            draws["state"] = r(N, 13)  # base_multirotor.py:182
            if self.spec.randomize_params:  # base_lee_controller.py:105-118 draws [k,3] per gain
                k = len(env_ids)
                for name in ("K_pos", "K_vel", "K_rot", "K_angvel"):
                    t = torch.zeros(N, 3, device=dev)
                    t[env_ids] = r(k, 3)
                    draws[name] = t
            draws["tau_inc"], draws["tau_dec"], draws["thrust"] = r(N, M), r(N, M), r(N, M)  # motor_model.py:140-150
            if self.spec.use_rps:
                draws["k_thrust"] = r(N, M)
            eng.reset(mask, draws)
        if saved_motors is not None:
            for k, t in saved_motors.items():
                getattr(eng, k)[env_ids] = t[env_ids]
        self._motors_initialised = True
        if self.articulated:
            # joint state: uniform in the joint_config ranges, drawn full-size on the device and selected by the mask (no host sync)
            D = eng.dof_state.shape[1]
            u = torch.rand(N, D, 2, device=dev)
            p0, p1, v0, v1 = self._dof_rng
            new = torch.stack([_lerp(p0, p1, u[..., 0]), _lerp(v0, v1, u[..., 1])], dim=-1)
            eng.dof_state.copy_(torch.where(mask.view(N, 1, 1), new, eng.dof_state))
        if self.sensor is not None and self.sensor_cfg.randomize_placement:  # warp_sensor.py:153-172
            k, S = len(env_ids), self.sensor_cfg.num_sensors
            t0, t1, e0, e1 = self._mount_rng
            self.sensor_mount[env_ids, :, 0:3] = _lerp(t0, t1, torch.rand(k, S, 3, device=dev))
            self.sensor_mount[env_ids, :, 3:7] = _quat_from_euler(_lerp(e0, e1, torch.rand(k, S, 3, device=dev)))
        if self.sensor is not None and self._sensor_link is not None:
            self._fold_link_into_mount()
        if self.imu is not None:
            self.imu.reset_idx(env_ids)
        eng.refresh()  # update_states of ALL envs (base_multirotor.py:204-205); sim_steps zeroed by the kernel
        self._update_body_state()

    def _update_body_state(self):
        if self._body_state is not None:
            self.engine.update_body_state()

    def _sample_assets_and_update_scene(self, env_ids, mask, A):
        gtd, dev = self.global_tensor_dict, self.device
        self._num_keep = self.keep_in_env
        self._reset_assets(env_ids, A)
        self._num_keep = self.keep_in_env // 2  # env_manager.py:285-295 (second, thinner sampling)
        samples = torch.bernoulli(0.15 * torch.ones(len(env_ids), device=dev))
        sel = torch.nonzero(samples).squeeze(-1)
        if len(sel) > 0:
            self._reset_assets(env_ids[sel], A // 2)
        self._num_keep = self.keep_in_env
        if self._obstacle_mass is not None:
            # free obstacles keep the twist the contact solve gave them: the reset writes the state ratios' zero velocities
            gtd["env_asset_state_tensor"][env_ids, :, 7:13] = 0.0
        if self.scene is not None:  # WarpEnv.reset_idx (warp_env_manager.py:40-54)
            idx = self._obj_asset.unsqueeze(-1).expand(-1, -1, 7)
            self._obj_pose.copy_(torch.gather(gtd["env_asset_state_tensor"][..., 0:7], 1, idx))
            self.scene.update(mask)

    def reset(self):
        self.reset_idx(torch.arange(self.num_envs, device=self.device))

    # ------------------------------------------------------------------------------------------
    # stepping (env_manager.py:328-432)
    # ------------------------------------------------------------------------------------------
    def reset_tensors(self):
        self.collision_tensor[:] = 0
        self.truncation_tensor[:] = 0

    def _draw_disturbance(self):
        """apply_disturbance (base_multirotor.py:213-234).  reset_rng = "torch": bernoulli, rand, rand in the reference's order.
        reset_rng = "device" (default): one launch of agx_disturbance_draw (Philox per env, keyed by the global env id and a draw
        counter) into a persistent [N,6] buffer -- same distributions, no torch RNG launches inside the physics loop."""
        sp, N, dev = self.spec, self.num_envs, self.device
        if not sp.enable_disturbance:
            return None
        if self.reset_rng == "device":
            if getattr(self, "_dist_buf", None) is None:
                self._dist_buf = torch.zeros(N, 6, device=dev)
                self._dist_max = (C.c_float * 6)(*[float(v) for v in sp.max_disturbance])
                self._dist_counter = 0
                self._dist_seed = (int(self.env_args.get("seed", 0)) ^ 0xD157_0000_D157) & (2**64 - 1)
            stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            _lib.check(_lib.load().agx_disturbance_draw(N, int(self.env_args.get("env_id_offset", 0)), float(sp.prob_apply_disturbance),
                                                        self._dist_max, self._dist_seed, self._dist_counter & 0xFFFFFFFF,
                                                        C.c_void_p(self._dist_buf.data_ptr()), stream), "agx_disturbance_draw")
            self._dist_counter += 1
            if self._dist_ctr_dev is not None:  # the graph path's device-resident copy of the counter follows
                _lib.check(_lib.load().agx_counter_add(C.c_void_p(self._dist_ctr_dev.data_ptr()), 1, stream), "agx_counter_add")
            return self._dist_buf
        occ = torch.bernoulli(sp.prob_apply_disturbance * torch.ones(N, device=dev))
        mx = torch.tensor(sp.max_disturbance, dtype=torch.float32, device=dev).expand(N, -1)
        f = _lerp(-mx[:, 0:3], mx[:, 0:3], torch.rand(N, 3, device=dev)) * occ.unsqueeze(1)
        t = _lerp(-mx[:, 3:6], mx[:, 3:6], torch.rand(N, 3, device=dev)) * occ.unsqueeze(1)
        return torch.cat([f, t], dim=1).contiguous()

    def _graph_for(self, n, moving=False):
        """CUDA graph of the n physics sub-steps of one env step (captured once per (n, moving)): per sub-step ONE physics launch that
        draws its disturbance in the kernel (AgxHp1Buffers.dist_counter: the draw counter lives in device memory, so a replay draws
        afresh) and ONE collision launch, then one single-thread kernel that advances the draw counter.  moving (contact with moving
        obstacles, an env step with env_actions): each sub-step begins with the obstacle advance and the scene re-pose, which read
        the persistent gtd["env_actions"].  Same kernels, same arithmetic, same draws as the launch-by-launch loop (tests:
        bit-identical trajectories); every C-ABI call is capture-safe (no allocation, no synchronisation).  Navigation-type envs run
        10 sub-steps per env step (config/env_config/env_with_obstacles.py:29-30): ~30 launches become one.
        Dynamic obstacles (args['contact_dynamic_obstacles'], fixed for the manager, so (n, moving) keys the graph): every sub-step
        advances the obstacles, with the env_actions twist when moving and with their own velocity otherwise, the solve writes the
        obstacles it pushes, and the scene is re-posed once more after the last sub-step.  With args['contact_obstacle_ground'] (also
        fixed for the manager) each sub-step's obstacle advance is followed by the obstacle-ground solve, and with
        args['contact_obstacle_obstacle'] (fixed too) by the obstacle-obstacle solve after it."""
        g = self._graphs.get((n, moving))
        if g is not None:
            return g
        eng, a = self.engine, self.global_tensor_dict["robot_actions"]
        dist = self.spec.enable_disturbance
        dynamic = self._obstacle_mass is not None
        if dist and self._dist_ctr_dev is None:
            self._draw_disturbance()  # creates the stream state (seed, counters); the draw itself is discarded ...
            self._dist_counter -= 1   # ... and not counted
            self._dist_ctr_dev = torch.tensor([self._dist_counter & 0xFFFFFFFF], dtype=torch.int32, device=self.device)
        lib = _lib.load()

        def body():
            for i in range(n):
                if moving or dynamic:
                    self._move_obstacles_one_substep(with_twist=moving)
                eng.physics_step(a, physics_steps=1, dist_counter=self._dist_ctr_dev if dist else None, dist_offset=i)
                self.compute_observations(moving_obstacles=moving or dynamic)
            if dynamic and n:
                self._repose_scene()
            if dist and n:
                _lib.check(lib.agx_counter_add(C.c_void_p(self._dist_ctr_dev.data_ptr()), n,
                                               C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)), "agx_counter_add")

        cur = torch.cuda.current_stream(self.device)
        side = torch.cuda.Stream(device=self.device)
        side.wait_stream(cur)
        with torch.cuda.stream(side):  # warm-up outside the capture (first launches may load modules), on throw-away copies of the state
            keep = (eng.root_state.clone(), eng.motor_thrust.clone(), self.collision_tensor.clone(),
                    None if not dist else self._dist_ctr_dev.clone())
            force = self.global_tensor_dict["robot_contact_force_tensor"]
            keep_force = force.clone()
            keep_dof = eng.dof_state.clone() if getattr(eng, "dof_state", None) is not None else None  # articulated robots
            if moving or dynamic:
                ast = self.global_tensor_dict["env_asset_state_tensor"]
                keep_obstacles = (ast.clone(), self._obj_pose.clone())
            body()
            eng.root_state.copy_(keep[0]); eng.motor_thrust.copy_(keep[1]); self.collision_tensor.copy_(keep[2])
            force.copy_(keep_force)
            if keep_dof is not None:
                eng.dof_state.copy_(keep_dof)
            if dist:
                self._dist_ctr_dev.copy_(keep[3])
            if moving or dynamic:
                ast.copy_(keep_obstacles[0]); self._obj_pose.copy_(keep_obstacles[1])
                self.scene.update()
        cur.wait_stream(side)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=side):
            body()
        # capturing does not execute: the state is untouched, the caller replays
        self._graphs[(n, moving)] = g
        return g

    def sample_physics_steps(self):
        e = self.cfg.env
        return max(math.floor(random.gauss(e.num_physics_steps_per_env_step_mean, e.num_physics_steps_per_env_step_std)), 0)

    def step(self, actions, env_actions=None):
        gtd = self.global_tensor_dict
        self.reset_tensors()
        if env_actions is not None:
            if self.num_obs_in_env > 1:
                want = (self.num_envs, self.num_obs_in_env, 6)
                if tuple(env_actions.shape) != want or env_actions.dtype != torch.float32 or env_actions.device.type != self.device.type:
                    raise ValueError(f"env_actions must be a float32 {list(want)} tensor on {self.device} (linear + angular velocity per obstacle)")
            if gtd["env_actions"] is None:
                # moving-obstacle contact replays graphs that read this buffer: it must be the manager's own, contiguous
                first = env_actions.contiguous().clone() if self._contact_motion is not None else env_actions
                gtd["env_actions"], gtd["prev_env_actions"] = first, env_actions.clone()
            gtd["prev_env_actions"][:] = gtd["env_actions"]
            gtd["env_actions"][:] = env_actions
        n = self.sample_physics_steps()
        gtd["robot_prev_actions"][:] = gtd["robot_actions"]  # robot_manager.py:486-488
        gtd["robot_actions"][:] = actions
        a = gtd["robot_actions"]
        obstacles_move = env_actions is not None and self.num_obs_in_env > 1
        # contact with moving obstacles: the obstacles advance inside each sub-step, before the robot's (the reference's order)
        moving = obstacles_move and self._contact_motion is not None
        # dynamic obstacles: free bodies that also drift (and get pushed) in steps without env_actions
        dynamic = self._obstacle_mass is not None
        if self.spec.enable_disturbance or self.scene is not None or self.contact_params is not None:
            # the reference loop (env_manager.py:426-428): fresh disturbance draws and a collision check (or contact solve) after
            # EVERY physics step
            if self.step_mode == "graph":
                self._graph_for(n, moving).replay()  # the n x (physics launch with in-kernel draw, collision launch) of this env step: one graph launch
                if self.spec.enable_disturbance:
                    self._dist_counter += n
            else:
                for i in range(n):
                    if moving or dynamic:
                        self._move_obstacles_one_substep(with_twist=moving)
                    self.engine.physics_step(a, disturbance=self._draw_disturbance(), physics_steps=1)
                    self.compute_observations(moving_obstacles=moving or dynamic)
                if dynamic and n:  # the solve moved the obstacles it pushed: sensors and the next step see them there
                    self._repose_scene()
        elif n > 0:
            self.engine.physics_step(a, physics_steps=n)  # n sub-steps fused in one launch
        if obstacles_move and not moving and n > 0:  # ObstacleManager.pre_physics_step, obstacle_manager.py:40-44
            self._step_obstacles(gtd["env_actions"], n)
        self._update_body_state()
        self.engine.sim_steps += 1
        self.step_counter += 1

    def simulate(self, actions, env_actions=None):
        """ONE physics step (env_manager.py:346-349: pre_physics_step -> physics -> post_physics_step), for callers that drive the loop
        themselves; step() batches the n physics steps of an env step into as few launches as the env allows"""
        gtd = self.global_tensor_dict
        gtd["robot_prev_actions"][:] = gtd["robot_actions"]
        gtd["robot_actions"][:] = actions
        self.engine.physics_step(gtd["robot_actions"], disturbance=self._draw_disturbance(), physics_steps=1)
        if env_actions is not None and self.num_obs_in_env > 1:
            self._step_obstacles(env_actions, 1)
        self._update_body_state()

    def render_viewer(self):
        return None  # headless by construction: there is no Isaac Gym viewer (env_manager.py:389-391)

    def log_memory_use(self):
        if self.device.type == "cuda":  # env_manager.py:303-326
            gb = 1024.0 ** 3
            print(f"torch.cuda.memory_allocated: {torch.cuda.memory_allocated(self.device) / gb:.3f} GB, "
                  f"reserved: {torch.cuda.memory_reserved(self.device) / gb:.3f} GB, max reserved: {torch.cuda.max_memory_reserved(self.device) / gb:.3f} GB")

    def _step_obstacles(self, twist, n):
        """dynamic_env: the obstacles' twist is overwritten with env_actions [N,A,6] before each of the n physics steps and
        the obstacles move (PhysX in the reference; agx_obstacle_step's kinematic advance here, one launch for the n steps).
        The reference leaves its Warp meshes stale until the next reset ("refit() ... expensive", env_manager.py:340-342);
        here re-posing + rebuilding the BVHs of all envs is one more launch, done by default (args['refit_dynamic_obstacles'])
        so the ray-cast sensors and the collision test of the next env step see the obstacles where they are."""
        self._advance_obstacles(twist, n)
        if self.scene is not None and bool(self.env_args.get("refit_dynamic_obstacles", True)):
            self._repose_scene()

    def _advance_obstacles(self, twist, n):
        gtd, N, A = self.global_tensor_dict, self.num_envs, self.num_obs_in_env
        ast = gtd["env_asset_state_tensor"]
        twist = twist.contiguous() if twist is not None else None  # shape / dtype / device were checked in step(); None: own velocity
        stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
        tw = C.c_void_p(twist.data_ptr()) if twist is not None else None
        _lib.check(_lib.load().agx_obstacle_step(N, A, C.c_void_p(ast.data_ptr()), ast.stride(1), tw,
                                                 float(self.sim_config.sim.dt), int(n), self._asset_damping[0], self._asset_damping[1],
                                                 stream), "agx_obstacle_step")

    def _repose_scene(self):
        idx = self._obj_asset.unsqueeze(-1).expand(-1, -1, 7)
        self._obj_pose.copy_(torch.gather(self.global_tensor_dict["env_asset_state_tensor"][..., 0:7], 1, idx))
        self.scene.update()

    def _move_obstacles_one_substep(self, with_twist=True):
        """contact with moving obstacles: one sub-step of the obstacles (the advance keeps its state in float32, so n of these add
        up bit for bit to one n-sub-step advance), with args['contact_obstacle_ground'] the obstacle-ground solve, with
        args['contact_obstacle_obstacle'] the obstacle-obstacle solve, and the scene re-posed where they now are.  with_twist False (dynamic obstacles in a step without env_actions): each obstacle keeps its own
        damped velocity."""
        self._advance_obstacles(self.global_tensor_dict["env_actions"] if with_twist else None, 1)
        if self._obstacle_hull is not None:  # obstacle-ground contact: the robot's contact search sees the corrected obstacles
            obstacle_ground_contact(self.contact_params, self._contact_motion, self._obstacle_mass, self._obstacle_hull)
        if self._obstacle_boxes is not None:  # obstacle-obstacle contact: after the ground's, so the scene shows both corrections
            obstacle_obstacle_contact(self.contact_params, self._contact_motion, self._obstacle_mass, self._obstacle_boxes)
        self._repose_scene()

    def compute_observations(self, moving_obstacles=False):
        """crashes += contact (env_manager.py:358-362).  PhysX contact forces are replaced by a
        geometric test: the base-link collision sphere overlaps the env mesh (agx_hp2_collide).  Contact mode: the contact solve
        (agx_hp2_contact) in its place, which flags by the contact force as the reference does.  moving_obstacles: the solve takes
        the obstacles' velocities (agx_hp2_contact_moving; only with args['contact_moving_obstacles']), and with
        args['contact_dynamic_obstacles'] also pushes them (agx_hp2_contact_dynamic)."""
        if self.contact_params is not None:
            hp2_contact(self.scene, self.engine.root_state, self.contact_params, self.global_tensor_dict["robot_contact_force_tensor"],
                        self.collision_tensor, motion=self._contact_motion if moving_obstacles else None,
                        mass=self._obstacle_mass if moving_obstacles else None)
        elif self.scene is not None:
            self.scene.collide(self.engine.root_state, self.robot.collision_radius, self.collision_tensor)

    def reset_terminated_and_truncated_envs(self):
        flags = self.collision_tensor * int(self.cfg.env.reset_on_collision) + self.truncation_tensor
        envs_to_reset = flags.nonzero(as_tuple=False).squeeze(-1)
        if len(envs_to_reset) > 0:
            self.reset_idx(envs_to_reset)
        return envs_to_reset

    def render(self, render_components="sensors"):
        if render_components == "sensors":
            self.render_sensors()

    def render_sensors(self):
        if self.imu is not None and self.articulated:
            # body b's force input of the last sub-step + m_b R_b^T g, R_b from its row of robot_body_state_tensor: the rigid path's
            # line below, per body
            fs, u = self.global_tensor_dict["force_sensor_tensor"], self.engine.imu_input
            fs[:, 0:3] = u[:, 0:3] + self._imu_mass.unsqueeze(1) * _quat_rotate_inverse(self.imu.robot_state[:, 3:7],
                                                                                          self.global_tensor_dict["gravity"])
            fs[:, 3:6] = u[:, 3:6]
            self._imu_angvel.copy_(u[:, 6:9])
            self.imu.update()
        elif self.imu is not None:
            gtd = self.global_tensor_dict
            fs, w = gtd["force_sensor_tensor"], self.engine.body_wrench
            fs[:, 0:3] = w[:, 0:3] + gtd["robot_mass"].unsqueeze(1) * _quat_rotate_inverse(gtd["robot_orientation"], gtd["gravity"])
            if self.contact_params is not None:  # PhysX's force sensor includes the contact force
                fs[:, 0:3] += _quat_rotate_inverse(gtd["robot_orientation"], gtd["robot_contact_force_tensor"])
            fs[:, 3:6] = w[:, 3:6]
            self.imu.update()
        if self.sensor is None:
            return
        self.sensor.capture()
        if self.sensor.noise_enabled:  # WarpSensor.apply_noise + apply_range_limits + normalize_observation (warp_sensor.py:197-250)
            if self._device_noise is not None:
                self._device_noise.apply()
            else:
                from ..sensors.noise import apply_noise_and_limits_torch
                apply_noise_and_limits_torch(self.global_tensor_dict["depth_range_pixels"], self.sensor_cfg)

    def post_reward_calculation_step(self):
        envs_to_reset = self.reset_terminated_and_truncated_envs()
        self.render(render_components="sensors")
        return envs_to_reset

    def get_obs(self):
        return self.global_tensor_dict

    def delete_env(self):
        if self.engine is not None:
            self.engine.close()
        self.engine = None
        self.scene = None
        self.sensor = None
