"""config/robot_config/{base_quad_config,base_quad_root_link_control_config,base_octarotor_config,
lmf1_config,lmf2_config,x500_config,magpie_config}.py -- the single-rigid-body multirotors.
Articulated robots (ROV, reconfigurable, Morphy) are out of the hot-path scope (SURVEY section 2 #21)."""
import numpy as np

from . import RESOURCES_DIRECTORY
from .sensor_config import (BaseDepthCameraConfig, BaseImuConfig, BaseLidarConfig, BaseLinkImuConfig, BaseNormalFaceIDCameraConfig,
                            GimbalCameraImuConfig, GimbalDepthCameraConfig, OSDome_64_Config, RSLidar_Airy_Config, StereoCameraConfig,
                            fake_radar_config, pmd_flexx2_config)

PI = np.pi
QUAD_ALLOCATION = [
    [0.0, 0.0, 0.0, 0.0],
    [0.0, 0.0, 0.0, 0.0],
    [1.0, 1.0, 1.0, 1.0],
    [-0.13, -0.13, 0.13, 0.13],
    [-0.13, 0.13, 0.13, -0.13],
    [-0.01, 0.01, -0.01, 0.01],
]


def _yaw_alloc(yaw_gain, plus_config=False):
    a = [row[:] for row in QUAD_ALLOCATION]
    if plus_config:  # lmf1 / x500 motor ordering
        a[3] = [-0.13, 0.13, 0.13, -0.13]
        a[4] = [-0.13, 0.13, -0.13, 0.13]
    a[5] = [-yaw_gain, yaw_gain, -yaw_gain, yaw_gain]
    return a


class BaseQuadCfg:
    class init_config:
        # [ratio_x, ratio_y, ratio_z, roll, pitch, yaw, 1.0, vx, vy, vz, wx, wy, wz]
        min_init_state = [0.1, 0.15, 0.15, 0, 0, -PI / 6, 1.0, -0.2, -0.2, -0.2, -0.2, -0.2, -0.2]
        max_init_state = [0.2, 0.85, 0.85, 0, 0, PI / 6, 1.0, 0.2, 0.2, 0.2, 0.2, 0.2, 0.2]

    class sensor_config:
        enable_camera = False
        camera_config = BaseDepthCameraConfig
        enable_lidar = False
        lidar_config = BaseLidarConfig
        enable_imu = False
        imu_config = BaseImuConfig

    class disturbance:
        enable_disturbance = False
        prob_apply_disturbance = 0.02
        max_force_and_torque_disturbance = [0.75, 0.75, 0.75, 0.004, 0.004, 0.004]

    class damping:
        linvel_linear_damping_coefficient = [0.0, 0.0, 0.0]
        linvel_quadratic_damping_coefficient = [0.0, 0.0, 0.0]
        angular_linear_damping_coefficient = [0.0, 0.0, 0.0]
        angular_quadratic_damping_coefficient = [0.0, 0.0, 0.0]

    class robot_asset:
        asset_folder = f"{RESOURCES_DIRECTORY}/robots/quad"
        file = "quad.urdf"
        name = "base_quadrotor"
        base_link_name = "base_link"
        disable_gravity = False
        collapse_fixed_joints = False
        fix_base_link = False
        collision_mask = 0
        replace_cylinder_with_capsule = False
        flip_visual_attachments = True
        density = 0.000001
        angular_damping = 0.01
        linear_damping = 0.01
        max_angular_velocity = 100.0
        max_linear_velocity = 100.0
        armature = 0.001
        semantic_id = 0
        per_link_semantic = False
        min_state_ratio = [0.1, 0.1, 0.1, 0, 0, -PI, 1.0, 0, 0, 0, 0, 0, 0]
        max_state_ratio = [0.3, 0.9, 0.9, 0, 0, PI, 1.0, 0, 0, 0, 0, 0, 0]
        max_force_and_torque_disturbance = [0.1, 0.1, 0.1, 0.05, 0.05, 0.05]
        color = None
        semantic_masked_links = {}
        keep_in_env = True
        min_position_ratio = None
        max_position_ratio = None
        min_euler_angles = [-PI, -PI, -PI]
        max_euler_angles = [PI, PI, PI]
        place_force_sensor = True
        force_sensor_parent_link = "base_link"
        force_sensor_transform = [0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0]
        use_collision_mesh_instead_of_visual = False

    class control_allocator_config:
        num_motors = 4
        force_application_level = "motor_link"  # or "root_link"
        application_mask = [1 + 4 + i for i in range(0, 4)]
        motor_directions = [1, -1, 1, -1]
        allocation_matrix = QUAD_ALLOCATION

        class motor_model_config:
            use_rps = True
            motor_thrust_constant_min = 0.00000926312
            motor_thrust_constant_max = 0.00001826312
            motor_time_constant_increasing_min = 0.04
            motor_time_constant_increasing_max = 0.04
            motor_time_constant_decreasing_min = 0.04
            motor_time_constant_decreasing_max = 0.04
            max_thrust = 2
            min_thrust = 0
            max_thrust_rate = 100000.0
            thrust_to_torque_ratio = 0.01
            use_discrete_approximation = True


class BaseQuadWithImuCfg(BaseQuadCfg):
    class sensor_config(BaseQuadCfg.sensor_config):
        enable_imu = True


class BaseQuadWithCameraCfg(BaseQuadCfg):
    class sensor_config(BaseQuadCfg.sensor_config):
        enable_camera = True


class BaseQuadWithCameraImuCfg(BaseQuadCfg):
    class sensor_config(BaseQuadCfg.sensor_config):
        enable_camera = True
        enable_imu = True


class BaseQuadWithLidarCfg(BaseQuadCfg):
    class sensor_config(BaseQuadCfg.sensor_config):
        enable_lidar = True


class BaseQuadWithFaceIDNormalCameraCfg(BaseQuadCfg):
    class sensor_config(BaseQuadCfg.sensor_config):
        enable_camera = True
        camera_config = BaseNormalFaceIDCameraConfig


class BaseQuadWithStereoCameraCfg(BaseQuadCfg):
    class sensor_config(BaseQuadCfg.sensor_config):
        enable_camera = True
        camera_config = StereoCameraConfig


class BaseQuadRootLinkControlCfg(BaseQuadCfg):
    class robot_asset(BaseQuadCfg.robot_asset):
        file = "model.urdf"

    class control_allocator_config(BaseQuadCfg.control_allocator_config):
        force_application_level = "root_link"

        class motor_model_config(BaseQuadCfg.control_allocator_config.motor_model_config):
            motor_thrust_constant_min = 0.00001826312
            motor_thrust_constant_max = 0.00001826312
            motor_time_constant_increasing_min = 0.01
            motor_time_constant_increasing_max = 0.03
            motor_time_constant_decreasing_min = 0.005
            motor_time_constant_decreasing_max = 0.005
            max_thrust = 10


class BaseOctarotorCfg(BaseQuadCfg):
    class init_config:
        min_init_state = [0.0, 0.0, 0.0, 0, 0, -PI, 1.0, -0.2, -0.2, -0.2, -0.2, -0.2, -0.2]
        max_init_state = [1.0, 1.0, 1.0, 0, 0, PI, 1.0, 0.2, 0.2, 0.2, 0.2, 0.2, 0.2]

    class disturbance:
        enable_disturbance = True
        prob_apply_disturbance = 0.05
        max_force_and_torque_disturbance = [1.5, 1.5, 1.5, 0.25, 0.25, 0.25]

    class robot_asset(BaseQuadCfg.robot_asset):
        asset_folder = f"{RESOURCES_DIRECTORY}/robots/octarotor"
        file = "octarotor.urdf"
        name = "base_octarotor"
        angular_damping = 0.0000001
        linear_damping = 0.0000001

    class control_allocator_config:
        num_motors = 8
        force_application_level = "motor_link"
        application_mask = [1 + 8 + i for i in range(0, 8)]
        motor_directions = [1, -1, 1, -1, 1, -1, 1, -1]
        allocation_matrix = [
            [-0.78867513, 0.21132487, -0.21132487, 0.78867513, 0.78867513, -0.21132487, 0.21132487, -0.78867513],
            [0.21132487, 0.78867513, -0.78867513, -0.21132487, -0.21132487, -0.78867513, 0.78867513, 0.21132487],
            [0.57735027, -0.57735027, -0.57735027, 0.57735027, 0.57735027, -0.57735027, -0.57735027, 0.57735027],
            [0.14226497, -0.21547005, 0.25773503, 0.01547005, -0.01547005, -0.25773503, 0.21547005, -0.14226497],
            [-0.25773503, 0.01547005, 0.14226497, 0.21547005, -0.21547005, -0.14226497, -0.01547005, 0.25773503],
            [0.11547005, -0.23094011, -0.11547005, 0.23094011, -0.23094011, 0.11547005, 0.23094011, -0.11547005],
        ]

        class motor_model_config:
            use_rps = False
            motor_thrust_constant_min = 0.00000926312
            motor_thrust_constant_max = 0.00001826312
            motor_time_constant_increasing_min = 0.01
            motor_time_constant_increasing_max = 0.03
            motor_time_constant_decreasing_min = 0.005
            motor_time_constant_decreasing_max = 0.005
            max_thrust = 6.25
            min_thrust = -6.25
            max_thrust_rate = 100000.0
            thrust_to_torque_ratio = 0.01
            use_discrete_approximation = True


class LMF2Cfg(BaseQuadCfg):
    class sensor_config(BaseQuadCfg.sensor_config):
        enable_camera = True
        lidar_config = pmd_flexx2_config  # lmf2_config.py:58 (disabled by default)

    class disturbance:
        enable_disturbance = True
        prob_apply_disturbance = 0.05
        max_force_and_torque_disturbance = [4.75, 4.75, 4.75, 0.03, 0.03, 0.03]

    class robot_asset(BaseQuadCfg.robot_asset):
        asset_folder = f"{RESOURCES_DIRECTORY}/robots/lmf2"
        file = "model.urdf"
        name = "base_quadrotor"
        collapse_fixed_joints = True
        max_state_ratio = [0.9, 0.9, 0.9, 0, 0, PI, 1.0, 0, 0, 0, 0, 0, 0]

    class control_allocator_config(BaseQuadCfg.control_allocator_config):
        force_application_level = "base_link"  # any non-"motor_link" string = wrench at body 0
        allocation_matrix = _yaw_alloc(0.07)

        class motor_model_config(BaseQuadCfg.control_allocator_config.motor_model_config):
            motor_time_constant_increasing_min = 0.05
            motor_time_constant_increasing_max = 0.08
            motor_time_constant_decreasing_min = 0.005
            motor_time_constant_decreasing_max = 0.005
            max_thrust = 10.0
            min_thrust = 0.1
            thrust_to_torque_ratio = 0.07


class MagpieCfg(LMF2Cfg):
    class init_config:
        min_init_state = [0.1, 0.15, 0.15, 0, 0, -PI, 1.0, -0.2, -0.2, -0.2, -0.2, -0.2, -0.2]
        max_init_state = [0.2, 0.85, 0.85, 0, 0, PI, 1.0, 0.2, 0.2, 0.2, 0.2, 0.2, 0.2]

    class sensor_config(BaseQuadCfg.sensor_config):
        enable_lidar = True
        lidar_config = RSLidar_Airy_Config  # magpie_config.py:52-53

    class robot_asset(BaseQuadCfg.robot_asset):
        asset_folder = f"{RESOURCES_DIRECTORY}/robots/magpie"
        file = "model.urdf"
        name = "base_quadrotor"
        collapse_fixed_joints = True
        max_state_ratio = [0.9, 0.9, 0.9, 0, 0, PI, 1.0, 0, 0, 0, 0, 0, 0]

    class control_allocator_config(LMF2Cfg.control_allocator_config):
        allocation_matrix = _yaw_alloc(0.02)

        class motor_model_config(BaseQuadCfg.control_allocator_config.motor_model_config):
            motor_time_constant_increasing_min = 0.01
            motor_time_constant_increasing_max = 0.02
            motor_time_constant_decreasing_min = 0.005
            motor_time_constant_decreasing_max = 0.015
            max_thrust = 12.0
            min_thrust = 0.1
            max_thrust_rate = 1000000.0
            thrust_to_torque_ratio = 0.02


class X500Cfg(BaseQuadCfg):
    class init_config:
        min_init_state = [0.0, 0.0, 0.0, -PI / 6, -PI / 6, -PI, 1.0, -0.5, -0.5, -0.5, -0.2, -0.2, -0.2]
        max_init_state = [1.0, 1.0, 1.0, PI / 6, PI / 6, PI, 1.0, 0.5, 0.5, 0.5, 0.2, 0.2, 0.2]

    class disturbance:
        enable_disturbance = False
        prob_apply_disturbance = 0.0
        max_force_and_torque_disturbance = [0, 0, 0, 0, 0, 0]

    class robot_asset(BaseQuadCfg.robot_asset):
        asset_folder = f"{RESOURCES_DIRECTORY}/robots/x500"
        file = "model.urdf"
        name = "base_quadrotor"
        collision_mask = 1
        armature = 0.00001
        max_state_ratio = [0.9, 0.9, 0.9, 0, 0, PI, 1.0, 0, 0, 0, 0, 0, 0]
        angular_damping = 0.02
        linear_damping = 0.02

    class control_allocator_config:
        num_motors = 4
        force_application_level = "motor_link"
        application_mask = [4, 1, 3, 2]
        motor_directions = [1, 1, -1, -1]
        allocation_matrix = _yaw_alloc(0.025, plus_config=True)

        class motor_model_config:
            use_rps = True
            motor_thrust_constant_min = 8.54858e-06
            motor_thrust_constant_max = 8.54858e-06
            motor_time_constant_increasing_min = 0.0125
            motor_time_constant_increasing_max = 0.0125
            motor_time_constant_decreasing_min = 0.025
            motor_time_constant_decreasing_max = 0.025
            max_thrust = 20.0
            min_thrust = 0.0
            max_thrust_rate = 100000.0
            thrust_to_torque_ratio = 0.025
            use_discrete_approximation = False


class LMF1Cfg(X500Cfg):
    class robot_asset(X500Cfg.robot_asset):
        asset_folder = f"{RESOURCES_DIRECTORY}/robots/lmf1"
        name = "base_quadrotor"

    class control_allocator_config(X500Cfg.control_allocator_config):
        allocation_matrix = _yaw_alloc(0.05, plus_config=True)

        class motor_model_config(X500Cfg.control_allocator_config.motor_model_config):
            motor_thrust_constant_min = 5.487e-06
            motor_thrust_constant_max = 5.487e-06
            motor_time_constant_increasing_min = 0.025
            motor_time_constant_increasing_max = 0.025
            thrust_to_torque_ratio = 0.05


class LMF2RadarCfg(LMF2Cfg):
    """config/robot_config/lmf2_radar_config.py: lmf2 with the 48 x 120 world-frame point-cloud "radar" instead of the camera"""
    class sensor_config(LMF2Cfg.sensor_config):
        enable_camera = False
        enable_lidar = True
        lidar_config = fake_radar_config


class TinyPropCfg(BaseQuadCfg):
    """config/robot_config/tinyprop_config.py (the sim2real end-to-end quadrotor)"""
    class init_config:
        min_init_state = [-0.7, -0.7, -0.7, -PI / 6, -PI / 6, -PI, 1.0, -0.5, -0.5, -0.5, -0.5, -0.5, -0.5]
        max_init_state = [0.7, 0.7, 0.7, PI / 6, PI / 6, PI, 1.0, 0.5, 0.5, 0.5, 0.5, 0.5, 0.5]

    class disturbance:
        enable_disturbance = False
        prob_apply_disturbance = 0.02
        max_force_and_torque_disturbance = [0.001, 0.001, 0.001, 0.00004, 0.00004, 0.00004]

    class robot_asset(BaseQuadCfg.robot_asset):
        asset_folder = f"{RESOURCES_DIRECTORY}/robots/tinyprop"
        file = "tinyprop.urdf"
        name = "tinyprop"

    class control_allocator_config(BaseQuadCfg.control_allocator_config):
        application_mask = [5, 6, 7, 8]
        allocation_matrix = [[0.0, 0.0, 0.0, 0.0], [0.0, 0.0, 0.0, 0.0], [1.0, 1.0, 1.0, 1.0], [-0.16, -0.16, 0.16, 0.16],
                             [-0.16, 0.16, 0.16, -0.16], [-0.01, 0.01, -0.01, 0.01]]

        class motor_model_config(BaseQuadCfg.control_allocator_config.motor_model_config):
            motor_thrust_constant_min = 0.00001286412
            motor_thrust_constant_max = 0.00001286412
            motor_time_constant_increasing_min = 0.047
            motor_time_constant_increasing_max = 0.047
            motor_time_constant_decreasing_min = 0.047
            motor_time_constant_decreasing_max = 0.047
            max_thrust = 1.2
            min_thrust = 0.2
            integration_scheme = "rk4"


class BaseRandCfg(BaseQuadCfg):
    """config/robot_config/base_random_config.py: an 8-rotor vehicle with arbitrarily placed, arbitrarily tilted rotors
    (resources/robots/random/random.urdf) -- the generic case of the per-link wrench map (SURVEY Appendix B)"""
    class init_config:
        min_init_state = [0.0, 0.0, 0.0, 0, 0, -PI, 1.0, -0.2, -0.2, -0.2, -0.2, -0.2, -0.2]
        max_init_state = [1.0, 1.0, 1.0, 0, 0, PI, 1.0, 0.2, 0.2, 0.2, 0.2, 0.2, 0.2]

    class disturbance:
        enable_disturbance = True
        prob_apply_disturbance = 0.05
        max_force_and_torque_disturbance = [1.5, 1.5, 1.5, 0.25, 0.25, 0.25]

    class robot_asset(BaseQuadCfg.robot_asset):
        asset_folder = f"{RESOURCES_DIRECTORY}/robots/random"
        file = "random.urdf"
        name = "base_random"
        angular_damping = 0.0000001
        linear_damping = 0.0000001
        min_state_ratio = [0.1, 0.1, 0.1, 0, 0, -PI, 1.0, -0.5, -0.5, -0.5, -0.2, -0.2, -0.2]
        max_state_ratio = [0.3, 0.9, 0.9, 0, 0, PI, 1.0, 0.5, 0.5, 0.5, 0.2, 0.2, 0.2]

    class control_allocator_config(BaseQuadCfg.control_allocator_config):
        num_motors = 8
        application_mask = [1 + 8 + i for i in range(0, 8)]
        motor_directions = [-1, 1, -1, 1, -1, 1, -1, 1]
        allocation_matrix = [
            [5.55111512e-17, -0.321393805, -0.454519478, -0.342020143, 0.96984631, 0.342020143, 0.866025404, -0.754406507],
            [1.0, -0.342020143, -0.707106781, 0.0, -0.173648178, 0.939692621, 0.5, -0.173648178],
            [1.66533454e-16, -0.883022222, 0.54167522, 0.939692621, 0.171010072, 1.11022302e-16, 1.11022302e-16, 0.633022222],
            [0.175, 0.123788742, -0.0569783368, 0.134977168, 0.0336959042, -0.266534135, -0.078839746, -0.0206893989],
            [0.01, 0.278845133, -0.0432852308, -0.272061766, -0.197793856, 0.0863687139, 0.156554446, -0.17126129],
            [0.282487373, -0.14173549, -0.0858541103, 0.0384858939, -0.333468026, 0.0836741468, 0.00846777988, -0.0874336259],
        ]

        class motor_model_config(BaseQuadCfg.control_allocator_config.motor_model_config):
            use_rps = False
            motor_time_constant_increasing_min = 0.01
            motor_time_constant_increasing_max = 0.03
            motor_time_constant_decreasing_min = 0.005
            motor_time_constant_decreasing_max = 0.005
            max_thrust = 5.0
            min_thrust = -5.0


class BaseROVCfg(BaseOctarotorCfg):
    """config/robot_config/base_rov_config.py: BlueROV2 with the octarotor's tilted-thruster allocation, no per-env gain randomisation
    on the robot side, disturbances on"""
    class init_config:
        min_init_state = [0.0, 0.0, 0.0, 0, 0, -PI, 1.0, -0.2, -0.2, -0.2, -0.2, -0.2, -0.2]
        max_init_state = [1.0, 1.0, 1.0, 0, 0, PI, 1.0, 0.2, 0.2, 0.2, 0.2, 0.2, 0.2]

    class disturbance:
        enable_disturbance = True
        prob_apply_disturbance = 0.05
        max_force_and_torque_disturbance = [1.5, 1.5, 1.5, 0.25, 0.25, 0.25]

    class robot_asset(BaseOctarotorCfg.robot_asset):
        asset_folder = f"{RESOURCES_DIRECTORY}/robots/BlueROV"
        file = "rov.urdf"
        name = "base_rov"


class MorphyStiffCfg(BaseQuadCfg):
    """config/robot_config/morphy_stiff_config.py: the Morphy airframe with its arm joints welded (every joint of morphy_stiff.urdf is
    fixed) -- a plain rigid quadrotor.  MorphyCompliantCfg below frees two joints per arm."""
    class init_config:
        min_init_state = [0.0, 0.0, 0.0, 0, 0, -PI / 6, 1.0, -0.2, -0.2, -0.2, -0.2, -0.2, -0.2]
        max_init_state = [1.0, 1.0, 1.0, 0, 0, PI / 6, 1.0, 0.2, 0.2, 0.2, 0.2, 0.2, 0.2]

    class disturbance(BaseQuadCfg.disturbance):
        enable_disturbance = True

    class robot_asset(BaseQuadCfg.robot_asset):
        asset_folder = f"{RESOURCES_DIRECTORY}/robots/morphy"
        file = "morphy_stiff.urdf"
        flip_visual_attachments = False

    class control_allocator_config(BaseQuadCfg.control_allocator_config):
        application_mask = [3, 6, 9, 12]
        allocation_matrix = [[0.0, 0.0, 0.0, 0.0], [0.0, 0.0, 0.0, 0.0], [1.0, 1.0, 1.0, 1.0], [-0.0785, -0.0785, 0.0785, 0.0785],
                             [-0.0785, 0.0785, 0.0785, -0.0785], [-0.01, 0.01, -0.01, 0.01]]

        class motor_model_config(BaseQuadCfg.control_allocator_config.motor_model_config):
            use_rps = False
            motor_time_constant_increasing_min = 0.01
            motor_time_constant_increasing_max = 0.03
            motor_time_constant_decreasing_min = 0.005
            motor_time_constant_decreasing_max = 0.005


class MorphyCompliantCfg(MorphyStiffCfg):
    """Morphy with compliant arms (ours: the reference's own morphy.urdf and config are not in this tree).  morphy_compliant.urdf is
    morphy_stiff.urdf with two revolute joints per arm: base_link_to_connecting_link_i sweeps the arm in the base plane,
    connecting_link_to_arm_motor_i flaps it up and down, both within +-0.6 rad.  The drive gains are OUR values, not Morphy's
    measured ones (DESIGN.md "Articulated robots" derives them): an arm's inertia about either joint is 0.01625 kg x (0.07 m)^2 =
    8.0e-5 kg m^2, so k = 1.0 N m / rad gives w = 112 rad/s and a hover flap deflection of ~0.05 rad, and d = 3.6e-3 N m s / rad a
    damping ratio of 0.2."""
    class robot_asset(MorphyStiffCfg.robot_asset):
        file = "morphy_compliant.urdf"

    class joint_config:
        # per DOF, in the order of the merged body table (sweep_0, flap_0, sweep_1, flap_1, ...); a scalar applies to all
        stiffness = 1.0
        damping = 3.6e-3
        # uniform reset ranges of the joint state (position rad, velocity rad/s)
        min_init_dof_position = -0.1
        max_init_dof_position = 0.1
        min_init_dof_velocity = 0.0
        max_init_dof_velocity = 0.0


class BaseQuadWithGimbalCameraCfg(BaseQuadCfg):
    """base_quadrotor with a two-axis camera gimbal (ours): quad_gimbal.urdf hangs gimbal_roll_joint (about x, +-0.8 rad) ->
    gimbal_pitch_joint (about y, [-0.8, 1.6] rad, +pi/2 looks straight down) -> gimbal_camera_link 6 cm below the base origin, and
    the 64 x 48 depth camera rides on gimbal_camera_link.  Each stage is balanced (COM on its axis), so the drive only has to move
    inertia: the roll subtree has 1.0e-5 kg m^2 about its axis, the pitch stage 6.0e-6.  With k = 0.03 N m / rad the drive's
    natural frequencies are 55 rad/s (roll) and 71 rad/s (pitch), w dt = 0.55 and 0.71 at dt = 0.01, and d = 7e-4 N m s / rad gives
    damping ratios of 0.64 and 0.82 (DESIGN.md "Articulated robots").  Targets (-roll, -pitch) of the base's ZYX Euler angles level
    the camera: Rz(psi) Ry(theta) Rx(phi) Rx(-phi) Ry(-theta) = Rz(psi)."""
    class sensor_config(BaseQuadCfg.sensor_config):
        enable_camera = True
        camera_config = GimbalDepthCameraConfig

    class robot_asset(BaseQuadCfg.robot_asset):
        file = "quad_gimbal.urdf"
        name = "base_quadrotor_with_gimbal_camera"

    class joint_config:
        # per DOF (gimbal_roll_joint, gimbal_pitch_joint); a scalar applies to both
        stiffness = 0.03
        damping = 7e-4
        min_init_dof_position = 0.0
        max_init_dof_position = 0.0
        min_init_dof_velocity = 0.0
        max_init_dof_velocity = 0.0


class BaseQuadWithGimbalCameraImuCfg(BaseQuadWithGimbalCameraCfg):
    """base_quadrotor_with_gimbal_camera with an IMU on gimbal_camera_link (GimbalCameraImuConfig): imu_measurement is the levelled
    camera's specific force and angular rate"""
    class sensor_config(BaseQuadWithGimbalCameraCfg.sensor_config):
        enable_imu = True
        imu_config = GimbalCameraImuConfig

    class robot_asset(BaseQuadWithGimbalCameraCfg.robot_asset):
        name = "base_quadrotor_with_gimbal_camera_imu"


class MorphyCompliantImuCfg(MorphyCompliantCfg):
    """morphy_compliant with an IMU on base_link: its force input includes the arms' joint reactions"""
    class sensor_config(MorphyCompliantCfg.sensor_config):
        enable_imu = True
        imu_config = BaseLinkImuConfig


class BaseQuadWithTorqueGimbalCfg(BaseQuadWithGimbalCameraCfg):
    """base_quadrotor_with_gimbal_camera with both gimbal joints in effort mode: no implicit drive, the commanded torques of
    dof_actuation_force_tensor [N, 2] (N m), each clamped to quad_gimbal.urdf's <limit effort> of 0.1 N m.  The camera still rides on
    gimbal_camera_link; levelling it is the caller's torque law (e.g. a PD on the base's Euler angles)."""
    class robot_asset(BaseQuadWithGimbalCameraCfg.robot_asset):
        name = "base_quadrotor_with_torque_gimbal"

    class joint_config(BaseQuadWithGimbalCameraCfg.joint_config):
        drive_mode = "effort"


class BaseQuadWithSlidingPayloadCfg(BaseQuadCfg):
    """base_quadrotor with a sliding payload (ours): quad_slider.urdf hangs payload_rail_joint, prismatic along the base x axis
    within +-0.05 m, 3 cm below the base origin, and payload_link (0.05 kg, COM on the rail) on it -- a moving-mass robot.  The drive
    acts on the relative motion of payload and airframe, whose reduced mass is mu = 0.05 x 0.25 / 0.30 = 0.042 kg: k = 10 N / m gives
    w = sqrt(k / mu) = 15.5 rad/s (w dt = 0.155 at dt = 0.01) and d = 0.9 N s / m a damping ratio d / (2 sqrt(k mu)) = 0.70
    (DESIGN.md "Articulated robots", "Prismatic joints").  Holding the payload at q* = 0.05 m takes m_p g q* = 0.025 N m of pitch
    torque: a thrust difference of 0.19 N across the motors' 0.13 m lever arm, 13 % of a motor pair's hover thrust."""
    class robot_asset(BaseQuadCfg.robot_asset):
        file = "quad_slider.urdf"
        name = "base_quadrotor_with_sliding_payload"

    class joint_config:
        # per DOF (payload_rail_joint: q in m, k in N / m, d in N s / m, drive_mode "effort" takes N); for a robot with several DOFs
        # a scalar applies to all and a list gives one value per DOF, each in its own joint's units
        stiffness = 10.0
        damping = 0.9
        min_init_dof_position = 0.0
        max_init_dof_position = 0.0
        min_init_dof_velocity = 0.0
        max_init_dof_velocity = 0.0
