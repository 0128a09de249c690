"""The host-side config mirror against the REFERENCE'S OWN config classes, field by field (this container only: the test
skips unless AERIAL_GYM_REFERENCE names a checkout of the reference).  Paths into the resource tree and the nested sensor config
classes of robot configs (compared on their own) are excluded; everything else must be equal."""
import importlib
import inspect
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
import _ref_loader  # noqa: E402

pytestmark = pytest.mark.skipif(not _ref_loader.reference_available(), reason="reference tree not present")

from aerial_gym_simulator_b200.config import (asset_config as AC, controller_config as CC, env_config as EC, robot_config as RC,  # noqa: E402
                                               sensor_config as S, sim_config as SC, task_config as TC)


def _flat(cls, prefix="", skip_nested=()):
    out = {}
    for k in dir(cls):
        if k.startswith("_") or k in skip_nested:
            continue
        v = getattr(cls, k)
        if inspect.isclass(v):
            out.update(_flat(v, prefix + k + ".", ()))
        elif not callable(v):
            out[prefix + k] = v
    return out


def _same(a, b):
    if isinstance(a, (str, bool, dict, type(None))) or isinstance(b, (str, type(None))):
        return a == b
    try:
        return np.array_equal(np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64))
    except (TypeError, ValueError):
        return a == b


def _compare(ref_cls, our_cls, skip=(), skip_nested=()):
    r, o = _flat(ref_cls, skip_nested=skip_nested), _flat(our_cls, skip_nested=skip_nested)
    assert len(r) >= 1
    bad = [(k, v, o.get(k, "<missing>")) for k, v in r.items() if not any(s in k for s in skip) and not _same(v, o.get(k, "<missing>"))]
    assert not bad, bad[:10]
    return len(r)


def _ref(mod, name):
    _ref_loader.install()
    return getattr(importlib.import_module("aerial_gym.config." + mod), name)


SENSORS = {
    "lidar_config.base_lidar_config": "BaseLidarConfig", "lidar_config.os0_128_config": "OS_0_128_Config",
    "lidar_config.os0_64_config": "OS_0_64_Config", "lidar_config.os1_64_config": "OS_1_64_Config", "lidar_config.os2_64_config": "OS_2_64_Config",
    "lidar_config.osdome_64_config": "OSDome_64_Config", "lidar_config.rslidar_airy_config": "RSLidar_Airy_Config",
    "lidar_config.pmd_flexx2_config": "pmd_flexx2_config", "lidar_config.st_vl53l5cx_config": "ST_VL53L5CXConfig",
    "lidar_config.fake_radar_config": "fake_radar_config", "camera_config.base_depth_camera_config": "BaseDepthCameraConfig",
    "camera_config.d455_depth_config": "RsD455Config", "camera_config.intel_realsense_d455_config": "IntelRealSenseD455Config",
    "camera_config.luxonis_oak_d_config": "LuxonisOakDConfig", "camera_config.luxonis_oak_d_pro_w_config": "LuxonisOakDProWConfig",
    "camera_config.stereo_camera_config": "StereoCameraConfig", "camera_config.base_normal_faceID_camera_config": "BaseNormalFaceIDCameraConfig",
    "imu_config.base_imu_config": "BaseImuConfig", "imu_config.bosch_bmi088_config": "BoschBMI088Config", "imu_config.vn100_config": "VN100Config",
}


@pytest.mark.parametrize("mod,name", sorted(SENSORS.items()))
def test_sensor_config(mod, name):
    _compare(_ref("sensor_config." + mod, name), getattr(S, name))


ROBOTS = {"morphy_stiff_config": "MorphyStiffCfg", "base_rov_config": "BaseROVCfg", "base_random_config": "BaseRandCfg", "tinyprop_config": "TinyPropCfg", "lmf2_radar_config": "LMF2RadarCfg", "base_quad_config": "BaseQuadCfg", "base_octarotor_config": "BaseOctarotorCfg", "lmf2_config": "LMF2Cfg", "magpie_config": "MagpieCfg",
          "x500_config": "X500Cfg", "lmf1_config": "LMF1Cfg", "base_quad_root_link_control_config": "BaseQuadRootLinkControlCfg"}


@pytest.mark.parametrize("mod,name", sorted(ROBOTS.items()))
def test_robot_config(mod, name):
    ref, ours = _ref("robot_config." + mod, name), getattr(RC, name)
    n = _compare(ref, ours, skip=("asset_folder",), skip_nested=("sensor_config",))
    assert n > 40
    rs, os_ = ref.sensor_config, ours.sensor_config  # which sensors are on, and which config class each one uses
    for k in ("enable_camera", "enable_lidar", "enable_imu"):
        assert getattr(rs, k) == getattr(os_, k), k
    for k in ("camera_config", "lidar_config", "imu_config"):
        assert getattr(rs, k).__name__ == getattr(os_, k).__name__, (k, getattr(rs, k).__name__, getattr(os_, k).__name__)


def test_controller_configs():
    for mod, name, ours in (("lee_controller_config", "control", CC.lee_controller_config),
                            ("lee_controller_config_octarotor", "control", CC.lee_controller_config_octarotor),
                            ("fully_actuated_controller_rov", "control", CC.fully_actuated_controller_config),
                            ("no_control_config", "control", CC.no_control_config),
                            ("lmf2_controller_config", "control", CC.lmf2_controller_config),
                            ("magpie_controller_config", "control", CC.magpie_controller_config)):
        _compare(_ref("controller_config." + mod, name), ours)


def test_env_sim_task_asset_configs():
    # (num_envs / use_warp are overwritten on the config CLASS by whoever built an env before, here as in the reference)
    _compare(_ref("env_config.empty_env", "EmptyEnvCfg"), EC.EmptyEnvCfg, skip=("asset_type_to_dict_map", "include_asset_type", "num_envs", "use_warp"))
    for mod, name, ours in (("env_with_obstacles", "EnvWithObstaclesCfg", EC.EnvWithObstaclesCfg),
                            ("env_with_lidar_nav_obstacles", "EnvWithLidarNavObstaclesCfg", EC.EnvWithLidarNavObstaclesCfg),
                            ("dynamic_environment", "DynamicEnvironmentCfg", EC.DynamicEnvironmentCfg), ("forest_env", "ForestEnvCfg", EC.ForestEnvCfg)):
        ref = _ref("env_config." + mod, name)
        _compare(ref.env, ours.env, skip=("num_envs", "use_warp"))
        assert ref.env_config.include_asset_type == ours.env_config.include_asset_type
        assert set(ref.env_config.asset_type_to_dict_map) == set(ours.env_config.asset_type_to_dict_map)
        for k in ref.env_config.asset_type_to_dict_map:  # every asset class of the map, switched on or not: all its parameters
            _compare(ref.env_config.asset_type_to_dict_map[k], ours.env_config.asset_type_to_dict_map[k], skip=("asset_folder",))
    for mod, name, ours in (("base_sim_config", "BaseSimConfig", SC.BaseSimConfig), ("base_sim_headless_config", "BaseSimHeadlessConfig", SC.BaseSimHeadlessConfig),
                            ("sim_config_2ms", "SimCfg2Ms", SC.SimCfg2Ms), ("sim_config_4ms", "SimCfg4Ms", SC.SimCfg4Ms),
                            ("custom_sim_config", "CustomSimConfig", SC.CustomSimConfig),
                            ("base_sim_no_gravity_config", "BaseSimNoGravityConfig", SC.BaseSimNoGravityConfig)):
        _compare(_ref("sim_config." + mod, name), ours)
    _compare(_ref("env_config.env_config_2ms", "EnvCfg2Ms"), EC.EnvCfg2Ms, skip=("asset_type_to_dict_map", "include_asset_type", "num_envs", "use_warp"))
    for name in ("BaseQuadWithImuCfg", "BaseQuadWithCameraCfg", "BaseQuadWithCameraImuCfg", "BaseQuadWithLidarCfg",
                 "BaseQuadWithFaceIDNormalCameraCfg", "BaseQuadWithStereoCameraCfg"):
        ref, ours = _ref("robot_config.base_quad_config", name), getattr(RC, name)
        for k in ("enable_camera", "enable_lidar", "enable_imu"):
            assert getattr(ref.sensor_config, k) == getattr(ours.sensor_config, k), (name, k)
        for k in ("camera_config", "lidar_config", "imu_config"):
            assert getattr(ref.sensor_config, k).__name__ == getattr(ours.sensor_config, k).__name__, (name, k)
    for mod, ours in (("position_setpoint_task_config", TC.position_setpoint_task_config), ("navigation_task_config", TC.navigation_task_config),
                      ("lidar_navigation_task_config", TC.lidar_navigation_task_config), ("radar_navigation_task_config", TC.radar_navigation_task_config),
                      ("position_setpoint_task_sim2real_config", TC.position_setpoint_task_sim2real_config),
                      ("position_setpoint_task_acceleration_sim2real_config", TC.position_setpoint_task_acceleration_sim2real_config)):
        _compare(_ref("task_config." + mod, "task_config"), ours, skip=("model_file", "model_folder", "headless", "device", "num_envs", "seed", "use_warp"))


def _all_paths():
    from aerial_gym_simulator_b200.compat_paths import CONFIG_MODULES
    return sorted((rel, name, where) for rel, names in CONFIG_MODULES.items() for name, where in names.items())


@pytest.mark.parametrize("rel,name,where", _all_paths())
def test_every_reference_config_path(rel, name, where):
    """compat_paths.CONFIG_MODULES: every (reference module path, name) resolves to a class here whose fields equal the reference
    class of THAT file (same-named asset classes differ between env_object_config / lidar_nav_env_config / dynamic_env_object_config)."""
    flat = {"sim_config": SC, "env_config": EC, "robot_config": RC, "controller_config": CC, "sensor_config": S, "asset_config": AC,
            "task_config": TC}
    mod_name, attr = where.split(".")
    ours, ref = getattr(flat[mod_name], attr), _ref(rel, name)
    assert inspect.isclass(ref) and inspect.isclass(ours)
    # resource paths differ by construction; num_envs / use_warp / seed / headless are overwritten on the class by whoever built an
    # env before; asset maps hold class objects (compared asset by asset in test_env_sim_task_asset_configs)
    skip = ("asset_folder", "num_envs", "use_warp", "seed", "headless", "asset_type_to_dict_map", "device", "vae_config.model_f")
    if name == "BaseEnvCfg":
        return  # an empty class on both sides
    _compare(ref, ours, skip=skip, skip_nested=("sensor_config",) if mod_name == "robot_config" else ())
