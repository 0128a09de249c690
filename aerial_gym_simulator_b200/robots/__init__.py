"""Robot registry surface (reference: aerial_gym/robots/__init__.py) for the single-rigid-body
multirotors; the robot object resolves configs + URDF into the flat MultirotorSpec the kernel takes."""
import os

import numpy as np

from .. import control  # noqa: F401  (registers controllers)
from .. import urdf
from ..config import robot_config as rc
from ..hp1 import ArticulationSpec, MultirotorSpec
from ..registry._core import controller_registry, robot_registry


class BaseMultirotor:
    """robots/base_multirotor.py + base_robot.py, construction half: owns no tensors (the engine
    does) and no arithmetic (the kernel does)."""

    def __init__(self, robot_config, controller_name, env_config, device):
        self.cfg = robot_config
        self.num_envs = env_config.env.num_envs
        self.device = device
        self.controller_name = controller_name
        self.controller, self.controller_config = controller_registry.make_controller(controller_name, self.num_envs, device)
        ca = self.cfg.control_allocator_config
        self.force_application_level = ca.force_application_level
        if controller_name == "no_control":
            self.controller_config.num_actions = ca.num_motors  # base_robot.py:33-34
        self.num_actions = self.controller_config.num_actions
        self.output_mode = "forces" if controller_name == "no_control" else "wrench"
        if self.force_application_level == "root_link" and controller_name == "no_control":
            raise ValueError("Force application level 'root_link' cannot be used with 'no_control'.")
        path = os.path.join(self.cfg.robot_asset.asset_folder, self.cfg.robot_asset.file)
        self.urdf_model = urdf.parse_urdf(path)
        self.robot_mass, self.robot_com, self.robot_inertia = self.urdf_model.composite_inertia()
        self.num_bodies = len(self.urdf_model.links)
        # collision proxy of body 0 (a14): bounding sphere of the root link's collision shapes
        root = self.urdf_model.links[self.urdf_model.root]
        rad = 0.0
        for c in root.collisions or root.visuals:
            ext = {"sphere": lambda v: v.size[0], "box": lambda v: 0.5 * float(np.linalg.norm(v.size)),
                   "cylinder": lambda v: float(np.hypot(v.size[0], 0.5 * v.size[1]))}.get(c.kind, lambda v: 0.0)(c)
            rad = max(rad, float(np.linalg.norm(c.p)) + ext)
        self.collision_radius = rad if rad > 0 else 0.1

    def make_spec(self, sim_config, env_config) -> MultirotorSpec:
        cfg, cc_, ca = self.cfg, self.controller_config, self.cfg.control_allocator_config
        mm = ca.motor_model_config
        M = ca.num_motors
        order, tf = self.urdf_model.body_order(), self.urdf_model.link_transforms()
        link_r, link_R = np.zeros((M, 3)), np.tile(np.eye(3), (M, 1, 1))
        if ca.force_application_level == "motor_link":
            for i, b in enumerate(ca.application_mask):
                if b >= len(order):
                    raise ValueError(f"application_mask entry {b} exceeds the {len(order)} bodies of the URDF")
                link_R[i], link_r[i] = tf[order[b]]
        g = lambda name, default: getattr(cc_, name, default)
        scheme = getattr(mm, "integration_scheme", "rk4")
        if scheme not in ("euler", "rk4"):
            scheme = "rk4"  # motor_model.py:13-19
        e = env_config.env
        return MultirotorSpec(
            num_motors=M, controller=self.controller.CONTROLLER_ID, dt=sim_config.sim.dt, gravity=tuple(sim_config.sim.gravity),
            mass=float(self.robot_mass), inertia=self.robot_inertia, com=self.robot_com,
            allocation_matrix=ca.allocation_matrix, motor_directions=ca.motor_directions,
            thrust_to_torque_ratio=mm.thrust_to_torque_ratio, force_application_level=ca.force_application_level,
            link_r=link_r, link_R=link_R, use_rps=bool(mm.use_rps), integration_scheme=scheme,
            use_discrete_approximation=bool(mm.use_discrete_approximation), min_thrust=float(mm.min_thrust),
            max_thrust=float(mm.max_thrust), max_thrust_rate=float(mm.max_thrust_rate),
            tau_inc_range=(mm.motor_time_constant_increasing_min, mm.motor_time_constant_increasing_max),
            tau_dec_range=(mm.motor_time_constant_decreasing_min, mm.motor_time_constant_decreasing_max),
            k_thrust_range=(mm.motor_thrust_constant_min, mm.motor_thrust_constant_max),
            max_yaw_rate=g("max_yaw_rate", np.pi / 3),
            K_pos_range=(tuple(g("K_pos_tensor_min", (0, 0, 0))), tuple(g("K_pos_tensor_max", (0, 0, 0)))),
            K_vel_range=(tuple(g("K_vel_tensor_min", (0, 0, 0))), tuple(g("K_vel_tensor_max", (0, 0, 0)))),
            K_rot_range=(tuple(g("K_rot_tensor_min", (0, 0, 0))), tuple(g("K_rot_tensor_max", (0, 0, 0)))),
            K_angvel_range=(tuple(g("K_angvel_tensor_min", (0, 0, 0))), tuple(g("K_angvel_tensor_max", (0, 0, 0)))),
            randomize_params=bool(g("randomize_params", False)),
            drag_lin1=tuple(cfg.damping.linvel_linear_damping_coefficient),
            drag_lin2=tuple(cfg.damping.linvel_quadratic_damping_coefficient),
            drag_ang1=tuple(cfg.damping.angular_linear_damping_coefficient),
            drag_ang2=tuple(cfg.damping.angular_quadratic_damping_coefficient),
            enable_disturbance=bool(cfg.disturbance.enable_disturbance),
            prob_apply_disturbance=float(cfg.disturbance.prob_apply_disturbance),
            max_disturbance=tuple(cfg.disturbance.max_force_and_torque_disturbance),
            linear_damping=float(cfg.robot_asset.linear_damping), angular_damping=float(cfg.robot_asset.angular_damping),
            max_linear_velocity=float(cfg.robot_asset.max_linear_velocity),
            max_angular_velocity=float(cfg.robot_asset.max_angular_velocity),
            min_init_state=tuple(cfg.init_config.min_init_state), max_init_state=tuple(cfg.init_config.max_init_state),
            bounds_lower_range=(tuple(e.lower_bound_min), tuple(e.lower_bound_max)),
            bounds_upper_range=(tuple(e.upper_bound_min), tuple(e.upper_bound_max)),
        )


class BaseROV(BaseMultirotor):
    """robots/base_rov.py: a fully actuated rigid body with eight thrusters (BlueROV2 geometry, gravity on, no buoyancy model in the
    reference either).  On the HP1 path it differs from BaseMultirotor in two bookkeeping points:
      * reset_idx does NOT touch the motor model (:188-201: no control_allocator.reset_idx) -- thrusts and time constants survive a
        reset; EnvManager.reset_idx restores them after the engine's reset (after the very first one, which stands in for
        MotorModel.init_tensors' initial draw);
      * robot_euler_angles is left in [0, 2 pi) (:245, no ssa).  Here the GTD tensor keeps the wrapped (-pi, pi] angles of the fused
        update_states; no controller of the ROV reads it (FullyActuatedController works on quaternions)."""
    keeps_motor_state_on_reset = True


class ArticulatedMultirotor(BaseMultirotor):
    """A multirotor whose URDF tree has revolute / continuous / prismatic joints (DESIGN.md "Articulated robots").  The controller, allocation and
    motor model are BaseMultirotor's, with the zero-configuration mass and inertia; the motors push on the bodies their links were
    merged into, and the joints are driven towards the engine's dof_position_setpoint / dof_velocity_setpoint by the drive of the
    config's joint_config (stiffness, damping per DOF; a scalar applies to every DOF).  joint_config.drive_mode ("position", the
    default, or "effort", per DOF or one for all) hands a DOF to the engine's dof_actuation_force instead, clamped to the URDF's
    <limit effort>.  Every DOF is in its joint's units: a revolute / continuous DOF in rad (k in N m / rad, d in N m s / rad, an
    effort in N m), a prismatic DOF in m (k in N / m, d in N s / m, an effort in N) -- in dof_state_tensor, the setpoints,
    dof_actuation_force_tensor and dof_force_tensor alike; a mixed robot gives its joint_config values as per-DOF lists."""
    articulated = True

    def __init__(self, robot_config, controller_name, env_config, device):
        super().__init__(robot_config, controller_name, env_config, device)
        if self.force_application_level != "motor_link":
            raise ValueError("an articulated robot needs force_application_level = 'motor_link': its motors push on the links "
                             "they belong to ('root_link' would apply them to the base)")
        self.bodies = self.urdf_model.articulation()  # raises for unsupported joints, zero axes and too many bodies

    def make_articulation(self) -> ArticulationSpec:
        ca, jc, b = self.cfg.control_allocator_config, self.cfg.joint_config, self.bodies
        order = self.urdf_model.body_order()
        M = ca.num_motors
        mb, mR, mp = np.zeros(M, np.int64), np.zeros((M, 3, 3)), np.zeros((M, 3))
        for i, idx in enumerate(ca.application_mask):
            if idx >= len(order):
                raise ValueError(f"application_mask entry {idx} exceeds the {len(order)} bodies of the URDF")
            link = order[idx]
            mb[i] = b.link_body[link]
            mR[i], mp[i] = b.link_in_body[link]
        cq = float(ca.motor_model_config.thrust_to_torque_ratio)
        return ArticulationSpec(
            bodies=b, stiffness=jc.stiffness, damping=jc.damping, motor_body=mb, motor_R=mR, motor_p=mp,
            motor_torque=-cq * np.asarray(ca.motor_directions, np.float64),
            init_dof_pos_range=(jc.min_init_dof_position, jc.max_init_dof_position),
            init_dof_vel_range=(jc.min_init_dof_velocity, jc.max_init_dof_velocity), drive_mode=getattr(jc, "drive_mode", "position"))


for _name, _cfg in (
    ("base_quadrotor", rc.BaseQuadCfg), ("base_octarotor", rc.BaseOctarotorCfg),
    ("base_quad_root_link_control", rc.BaseQuadRootLinkControlCfg), ("lmf1", rc.LMF1Cfg), ("lmf2", rc.LMF2Cfg),
    ("x500", rc.X500Cfg), ("magpie", rc.MagpieCfg), ("base_quadrotor_with_imu", rc.BaseQuadWithImuCfg),
    ("base_quadrotor_with_camera", rc.BaseQuadWithCameraCfg), ("base_quadrotor_with_camera_imu", rc.BaseQuadWithCameraImuCfg),
    ("base_quadrotor_with_lidar", rc.BaseQuadWithLidarCfg),
    ("base_quadrotor_with_faceid_normal_camera", rc.BaseQuadWithFaceIDNormalCameraCfg),
    ("base_quadrotor_with_stereo_camera", rc.BaseQuadWithStereoCameraCfg), ("lmf2_radar", rc.LMF2RadarCfg), ("tinyprop", rc.TinyPropCfg), ("base_random", rc.BaseRandCfg), ("morphy_stiff", rc.MorphyStiffCfg),
):
    robot_registry.register(_name, BaseMultirotor, _cfg)
robot_registry.register("base_rov", BaseROV, rc.BaseROVCfg)
robot_registry.register("morphy_compliant", ArticulatedMultirotor, rc.MorphyCompliantCfg)
robot_registry.register("base_quadrotor_with_gimbal_camera", ArticulatedMultirotor, rc.BaseQuadWithGimbalCameraCfg)
robot_registry.register("base_quadrotor_with_gimbal_camera_imu", ArticulatedMultirotor, rc.BaseQuadWithGimbalCameraImuCfg)
robot_registry.register("morphy_compliant_imu", ArticulatedMultirotor, rc.MorphyCompliantImuCfg)
robot_registry.register("base_quadrotor_with_torque_gimbal", ArticulatedMultirotor, rc.BaseQuadWithTorqueGimbalCfg)
robot_registry.register("base_quadrotor_with_sliding_payload", ArticulatedMultirotor, rc.BaseQuadWithSlidingPayloadCfg)

# the reference's package also exports its robot config classes (robots/__init__.py: `from ...base_quad_config import *`, ...)
globals().update({_k: _v for _k, _v in vars(rc).items() if _k.endswith("Cfg")})
