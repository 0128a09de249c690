"""config/sensor_config/{base_sensor_config, camera_config/base_depth_camera_config,
lidar_config/{base_lidar_config,osdome_64_config}}.py"""


class BaseSensorConfig:
    num_sensors = 1
    randomize_placement = False
    min_translation = [0.07, -0.06, 0.01]
    max_translation = [0.12, 0.03, 0.04]
    min_euler_rotation_deg = [-5.0, -5.0, -5.0]
    max_euler_rotation_deg = [5.0, 5.0, 5.0]


class BaseDepthCameraConfig(BaseSensorConfig):
    num_sensors = 1
    sensor_type = "camera"
    height, width = 135, 240
    horizontal_fov_deg = 87.000
    max_range, min_range = 10.0, 0.2
    calculate_depth = True  # depth image; False -> range image
    return_pointcloud = False
    pointcloud_in_world_frame = False
    segmentation_camera = True
    euler_frame_rot_deg = [-90.0, 0, -90.0]  # optical axis (+z) onto robot +x
    normalize_range = True
    far_out_of_range_value = max_range if normalize_range else -1.0
    near_out_of_range_value = -max_range if normalize_range else -1.0
    randomize_placement = True
    nominal_position = [0.10, 0.0, 0.03]
    nominal_orientation_euler_deg = [0.0, 0.0, 0.0]
    use_collision_geometry = False

    class sensor_noise:
        enable_sensor_noise = False
        pixel_dropout_prob = 0.01
        pixel_std_dev_multiplier = 0.01


class GimbalDepthCameraConfig(BaseDepthCameraConfig):
    """64 x 48 depth + segmentation camera on gimbal_camera_link of quad_gimbal.urdf (ours): parent_link makes EnvManager take the
    camera's pose from that link's body row of robot_body_state_tensor; the optical axis is the link's +x; fixed placement."""
    height, width = 48, 64
    parent_link = "gimbal_camera_link"
    randomize_placement = False
    min_translation = [0.0, 0.0, 0.0]
    max_translation = [0.0, 0.0, 0.0]
    min_euler_rotation_deg = [0.0, 0.0, 0.0]
    max_euler_rotation_deg = [0.0, 0.0, 0.0]


class BaseLidarConfig(BaseSensorConfig):
    num_sensors = 1
    sensor_type = "lidar"
    height, width = 128, 512
    horizontal_fov_deg_min, horizontal_fov_deg_max = -180, 180
    vertical_fov_deg_min, vertical_fov_deg_max = -45, +45
    max_range, min_range = 10.0, 0.2
    return_pointcloud = False
    pointcloud_in_world_frame = False
    segmentation_camera = True
    euler_frame_rot_deg = [0.0, 0.0, 0.0]
    normalize_range = True
    far_out_of_range_value = max_range if normalize_range else -1.0
    near_out_of_range_value = -max_range if normalize_range else -1.0
    randomize_placement = True
    nominal_position = [0.10, 0.0, 0.03]
    nominal_orientation_euler_deg = [0.0, 0.0, 0.0]

    class sensor_noise:
        enable_sensor_noise = True
        std_a = 0.00001
        std_b = 0.00001
        std_c = 0.00001
        mean_offset = -0.05
        pixel_dropout_prob = 0.0


class OSDome_64_Config(BaseLidarConfig):
    height, width = 64, 512
    vertical_fov_deg_min, vertical_fov_deg_max = 0, 90
    max_range, min_range = 20.0, 0.5
    # quirk kept: far/near_out_of_range_value are inherited from BaseLidarConfig (computed with ITS
    # max_range = 10), so an out-of-range return normalises to 10/20 = 0.5 (osdome_64_config.py:4-13)
    randomize_placement = False
    min_translation = [0.0, 0.0, 0.0]
    max_translation = [0.0, 0.0, 0.0]
    min_euler_rotation_deg = [0.0, 0.0, 0.0]
    max_euler_rotation_deg = [0.0, 0.0, 0.0]

    class sensor_noise:
        enable_sensor_noise = False
        std_a = 0.00038089
        std_b = -0.00343351
        std_c = 0.01553284
        mean_offset = -0.025
        pixel_dropout_prob = 0.0


class RSLidar_Airy_Config(BaseLidarConfig):
    """config/sensor_config/lidar_config/rslidar_airy_config.py: 48 x 120 hemispherical LiDAR that returns a WORLD-frame
    point cloud (what LiDARNavigationTask.process_image_observation consumes)."""
    height, width = 48, 120
    vertical_fov_deg_min, vertical_fov_deg_max = 0, 90
    max_range, min_range = 10.0, 0.2
    return_pointcloud = True
    segmentation_camera = False
    normalize_range = False
    pointcloud_in_world_frame = True
    randomize_placement = True  # a degenerate range: the mount is fixed, but the draws are still made
    min_translation = [-0.05, 0.0, 0.0]
    max_translation = [-0.05, 0.0, 0.0]
    min_euler_rotation_deg = [0.0, -90.0, 0.0]
    max_euler_rotation_deg = [0.0, -90.0, 0.0]

    class sensor_noise:
        enable_sensor_noise = False
        std_a = 0.00038089
        std_b = -0.00343351
        std_c = 0.01553284
        mean_offset = -0.025
        pixel_dropout_prob = 0.0


class DepthCamera64x48Config(BaseDepthCameraConfig):
    """BASELINE.json north-star sensor: 64x48 depth + segmentation."""
    height, width = 48, 64


# ---- the rest of the reference's sensor catalogue (config/sensor_config/{lidar,camera,imu}_config/*.py).  Unlike OSDome_64_Config
# these files recompute far / near_out_of_range_value from their OWN max_range.
def _noise(std_a, std_b, std_c, mean_offset, dropout, enabled=False):
    return type("sensor_noise", (), dict(enable_sensor_noise=enabled, std_a=std_a, std_b=std_b, std_c=std_c, mean_offset=mean_offset,
                                         pixel_dropout_prob=dropout))


def _ranged(base, name, doc, **kw):
    """subclass with far / near values derived from the class's own max_range and normalize_range, as the reference files do"""
    cls = type(name, (base,), dict(kw, __doc__=doc))
    if cls.return_pointcloud and cls.pointcloud_in_world_frame:
        cls.normalize_range = False
    cls.far_out_of_range_value = cls.max_range if cls.normalize_range else -1.0
    cls.near_out_of_range_value = -cls.max_range if cls.normalize_range else -1.0
    return cls


OS_0_128_Config = _ranged(BaseLidarConfig, "OS_0_128_Config", "lidar_config/os0_128_config.py", height=128, width=512, max_range=35.0,
                          min_range=0.2, sensor_noise=_noise(3.36239104e-05, -3.17199061e-04, 9.61903860e-03, -0.05, 0.0))
OS_0_64_Config = _ranged(OS_0_128_Config, "OS_0_64_Config", "lidar_config/os0_64_config.py", height=64,
                         sensor_noise=_noise(3.36239104e-05, -3.17199061e-04, 9.61903860e-03, -0.025, 0.0))
# quirk kept: OS-1 / OS-2 only override max_range; far / near values stay those of OS_0_128_Config (35 m)  (os1_64_config.py:4-14)
OS_1_64_Config = type("OS_1_64_Config", (OS_0_128_Config,), dict(
    __doc__="lidar_config/os1_64_config.py", height=64, vertical_fov_deg_min=-22.5, vertical_fov_deg_max=22.5, max_range=90.0, min_range=0.7,
    sensor_noise=_noise(3.08287454e-06, -4.07347360e-06, 5.30757302e-03, -0.025, 0.0)))
OS_2_64_Config = type("OS_2_64_Config", (OS_0_128_Config,), dict(
    __doc__="lidar_config/os2_64_config.py", height=64, vertical_fov_deg_min=-11.25, vertical_fov_deg_max=11.25, max_range=200.0, min_range=0.7,
    sensor_noise=_noise(3.08287454e-06, -4.07347360e-06, 5.30757302e-03, -0.025, 0.0)))
_TOF_MOUNT = dict(min_translation=[0.07, -0.06, 0.02], max_translation=[0.12, 0.03, 0.06], min_euler_rotation_deg=[-5.0, -5.0, -5.0],
                  max_euler_rotation_deg=[5.0, 5.0, 5.0])
pmd_flexx2_config = _ranged(BaseLidarConfig, "pmd_flexx2_config", "lidar_config/pmd_flexx2_config.py", height=172, width=224,
                            horizontal_fov_deg_min=-28, horizontal_fov_deg_max=28, vertical_fov_deg_min=-22, vertical_fov_deg_max=22,
                            max_range=5.0, min_range=0.2, segmentation_camera=False, randomize_placement=True,
                            sensor_noise=_noise(3.08287454e-06, -4.07347360e-06, 5.30757302e-03, -0.025, 0.01), **_TOF_MOUNT)
ST_VL53L5CXConfig = _ranged(BaseLidarConfig, "ST_VL53L5CXConfig", "lidar_config/st_vl53l5cx_config.py", height=8, width=8,
                            horizontal_fov_deg_min=-45, horizontal_fov_deg_max=45, vertical_fov_deg_min=-45, vertical_fov_deg_max=45,
                            max_range=4.0, min_range=0.2, segmentation_camera=False, normalize_range=False, randomize_placement=False,
                            min_translation=[0.07, -0.06, 0.01], max_translation=[0.12, 0.03, 0.04],
                            sensor_noise=_noise(3.08287454e-06, -4.07347360e-06, 5.30757302e-03, -0.025, 0.0))
fake_radar_config = _ranged(BaseLidarConfig, "fake_radar_config", "lidar_config/fake_radar_config.py (radar_navigation_task's sensor)",
                            height=48, width=120, horizontal_fov_deg_min=-60, horizontal_fov_deg_max=60, vertical_fov_deg_min=-60,
                            vertical_fov_deg_max=60, max_range=10.0, min_range=0.2, return_pointcloud=True, pointcloud_in_world_frame=True,
                            segmentation_camera=False, normalize_range=False, randomize_placement=True,
                            sensor_noise=_noise(3.08287454e-06, -4.07347360e-06, 5.30757302e-03, -0.025, 0.01), **_TOF_MOUNT)
_CAM_MOUNT = dict(min_translation=[0.07, -0.06, 0.01], max_translation=[0.12, 0.03, 0.04], min_euler_rotation_deg=[-5.0, -5.0, -5.0],
                  max_euler_rotation_deg=[5.0, 5.0, 5.0])
RsD455Config = _ranged(BaseDepthCameraConfig, "RsD455Config", "camera_config/d455_depth_config.py", height=270, width=480, max_range=15.0,
                       min_range=0.2, randomize_placement=True, **_CAM_MOUNT)
IntelRealSenseD455Config = _ranged(BaseDepthCameraConfig, "IntelRealSenseD455Config", "camera_config/intel_realsense_d455_config.py",
                                   height=270, width=480, max_range=15.0, min_range=0.2, randomize_placement=True, **_CAM_MOUNT)
LuxonisOakDConfig = _ranged(BaseDepthCameraConfig, "LuxonisOakDConfig", "camera_config/luxonis_oak_d_config.py", height=270, width=480,
                            horizontal_fov_deg=72.0, max_range=12.0, min_range=0.7, segmentation_camera=False, randomize_placement=False,
                            **_CAM_MOUNT)
# quirk kept: only the scalar fields are overridden, far / near values stay LuxonisOakDConfig's  (luxonis_oak_d_pro_w_config.py)
LuxonisOakDProWConfig = type("LuxonisOakDProWConfig", (LuxonisOakDConfig,), dict(
    __doc__="camera_config/luxonis_oak_d_pro_w_config.py", horizontal_fov_deg=127.0, max_range=12.0, min_range=0.2))
StereoCameraConfig = type("StereoCameraConfig", (BaseDepthCameraConfig,), dict(
    __doc__="camera_config/stereo_camera_config.py", sensor_type="stereo_camera", height=270, width=480, baseline=-0.095))
BaseNormalFaceIDCameraConfig = type("BaseNormalFaceIDCameraConfig", (BaseDepthCameraConfig,), dict(
    __doc__="camera_config/base_normal_faceID_camera_config.py", sensor_type="normal_faceID_camera", height=270, width=480,
    return_pointcloud=True, normal_in_world_frame=True, randomize_placement=False, **_CAM_MOUNT))


class BaseImuConfig(BaseSensorConfig):
    """config/sensor_config/imu_config/base_imu_config.py (values of a sample VN100)."""
    num_sensors = 1
    sensor_type = "imu"
    world_frame = False
    enable_noise = True
    enable_bias = True
    bias_std = [9.782812831313576e-07] * 3 + [2.6541629581345176e-05] * 3          # accel x3, gyro x3
    imu_noise_std = [0.001688956233495657] * 3 + [0.0010679343003532472] * 3
    max_measurement_value = [100.0, 100.0, 100.0, 10.0, 10.0, 10.0]
    max_bias_init_value = [1.0e-03] * 6
    gravity_compensation = False
    randomize_placement = False
    min_euler_rotation_deg = [-2.0, -2.0, -2.0]
    max_euler_rotation_deg = [2.0, 2.0, 2.0]


class BaseLinkImuConfig(BaseImuConfig):
    """an IMU on base_link (ours): on an articulated robot an IMU names its link; its force input is the base body's, the arms'
    joint reactions included"""
    parent_link = "base_link"


class GimbalCameraImuConfig(BaseImuConfig):
    """an IMU on gimbal_camera_link of quad_gimbal.urdf (ours), next to the gimbal's camera: parent_link makes EnvManager read the
    force, orientation and angular velocity of that link's body (the gimbal's pitch stage), so the IMU measures what the levelled
    camera feels, as a gimbal controller's own IMU does"""
    parent_link = "gimbal_camera_link"


class BoschBMI088Config(BaseImuConfig):
    """imu_config/bosch_bmi088_config.py"""
    bias_std = [0.0013564659966250536] * 3 + [1.4352700094407325e-05] * 3
    imu_noise_std = [0.0015690639999999998, 0.0015690639999999998, 0.0018632634999999997] + [0.0002443460952792061] * 3
    randomize_placement = True


class VN100Config(BaseImuConfig):
    """imu_config/vn100_config.py"""
    imu_noise_std = [0.001372931] * 3 + [6.108652381980153e-05] * 3
    randomize_placement = True
