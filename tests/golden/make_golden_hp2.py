"""HP2 fixtures produced by RUNNING THE REFERENCE'S OWN SENSOR CODE (this container only):

    python tests/golden/make_golden_hp2.py

The reference's `WarpSensor` (sensors/warp/warp_sensor.py) with its `WarpCam` / `WarpLidar` / `WarpStereoCam` / `WarpNormalFaceID*`
classes and every `@wp.kernel` they launch are imported UNMODIFIED from $AERIAL_GYM_REFERENCE; `warp` itself (warp-lang 1.0.0, not
installable) is the interpreter stub of tests/golden/_warp_stub.py, whose one stand-in is the mesh query (brute-force closest hit).
Pinned by these fixtures (SURVEY 8 rows b1-b7): camera matrices and LiDAR ray table (b6), sensor pose composition (b7), ray
generation, depth-vs-range multiplier, far plane, miss values, segmentation lookup, point-cloud and normal frames, stereo logic
(b1-b5), range limits and normalisation (b7).  NOT pinned: Warp's BVH traversal / tie-breaking (b9) and device rounding -- the
interpreter is fp32 without FMA contraction, so consumers compare depths to a tolerance and segmentation ids away from silhouette
edges (tests/test_hp2_reference_fixtures.py)."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import _ref_loader  # noqa: E402
import _warp_stub  # noqa: E402

_ref_loader.install()
_warp_stub.install()

from aerial_gym.sensors.warp.warp_sensor import WarpSensor  # noqa: E402
from aerial_gym.config.sensor_config.camera_config.base_depth_camera_config import BaseDepthCameraConfig  # noqa: E402
from aerial_gym.config.sensor_config.camera_config.stereo_camera_config import StereoCameraConfig  # noqa: E402
from aerial_gym.config.sensor_config.camera_config.base_normal_faceID_camera_config import BaseNormalFaceIDCameraConfig  # noqa: E402
from aerial_gym.config.sensor_config.lidar_config.osdome_64_config import OSDome_64_Config  # noqa: E402
from aerial_gym.config.sensor_config.lidar_config.rslidar_airy_config import RSLidar_Airy_Config  # noqa: E402
try:
    from aerial_gym.config.sensor_config.lidar_config.base_normal_faceID_lidar_config import BaseNormalFaceIDLidarConfig  # noqa: E402
except Exception:  # noqa: BLE001
    BaseNormalFaceIDLidarConfig = None

# the sensor classes default to device="cuda:0" and WarpSensor does not pass its own device on: the one substitution made here
import aerial_gym.sensors.warp.warp_sensor as _ws_mod  # noqa: E402
for _n in ("WarpCam", "WarpStereoCam", "WarpLidar", "WarpNormalFaceIDCam", "WarpNormalFaceIDLidar"):
    _c = getattr(_ws_mod, _n)
    _c.__init__.__defaults__ = tuple("cpu" if d == "cuda:0" else d for d in (_c.__init__.__defaults__ or ()))

from tests import _hp2_common as H  # noqa: E402  (scene builder shared with the consumers: same triangles on both sides)

E, K = 3, 14


class _NoNoise:
    enable_sensor_noise = False
    pixel_dropout_prob = 0.0
    pixel_std_dev_multiplier = 0.0


def variant(base, **kw):
    kw.setdefault("sensor_noise", _NoNoise)
    kw.setdefault("randomize_placement", False)
    return type("Cfg", (base,), kw)


CASES = {
    # name: (reference config class, overrides)
    "cam_depth_seg": (BaseDepthCameraConfig, dict(height=12, width=20, segmentation_camera=True)),
    "cam_range_noseg": (BaseDepthCameraConfig, dict(height=12, width=20, calculate_depth=False, segmentation_camera=False)),
    "cam_pc_sensor_seg": (BaseDepthCameraConfig, dict(height=10, width=14, return_pointcloud=True, pointcloud_in_world_frame=False, segmentation_camera=True)),
    "cam_pc_world": (BaseDepthCameraConfig, dict(height=10, width=14, return_pointcloud=True, pointcloud_in_world_frame=True, segmentation_camera=False,
                                                 normalize_range=False)),
    "lidar_range_seg": (OSDome_64_Config, dict(height=8, width=24)),
    "lidar_pc_world": (RSLidar_Airy_Config, dict(height=6, width=20)),
    "stereo_depth": (StereoCameraConfig, dict(height=10, width=16)),
    "normal_faceid_cam": (BaseNormalFaceIDCameraConfig, dict(height=10, width=14)),
}
if BaseNormalFaceIDLidarConfig is not None:
    CASES["normal_faceid_lidar"] = (BaseNormalFaceIDLidarConfig, dict(height=6, width=20))

FIELDS = ["sensor_type", "num_sensors", "height", "width", "horizontal_fov_deg", "horizontal_fov_deg_min", "horizontal_fov_deg_max",
          "vertical_fov_deg_min", "vertical_fov_deg_max", "max_range", "min_range", "calculate_depth", "return_pointcloud",
          "pointcloud_in_world_frame", "segmentation_camera", "normalize_range", "far_out_of_range_value", "near_out_of_range_value",
          "euler_frame_rot_deg", "baseline", "normal_in_world_frame"]


def main():
    sc = H.make_scene(E, K, seed=21, extent=2.2)
    tris, segs, cnt = H.oracle_tris(sc)  # world-space triangles [E, 12K, 9] and their segmentation ids (oracle/hp2_oracle.c: build_world_tris)
    meshes = []
    for e in range(E):
        t9 = tris[e]  # oracle layout: (v0, e1 = v1 - v0, e2 = v2 - v0) per triangle
        pts = np.stack([t9[:, 0:3], t9[:, 0:3] + t9[:, 3:6], t9[:, 0:3] + t9[:, 6:9]], axis=1).reshape(-1, 3)
        vel = np.zeros_like(pts)
        vel[:, 0] = np.repeat(segs[e], 3)  # seg id in the x component of every vertex' "velocity" (warp_env_manager.py:76-80)
        meshes.append(_warp_stub.Mesh(pts, np.arange(pts.shape[0], dtype=np.int32), vel))
    out = {"tris": tris, "segs": segs, "tri_count": cnt, "scene_seed": np.array(21), "E": np.array(E), "K": np.array(K)}
    g = torch.Generator().manual_seed(5)
    robot = torch.zeros(E, 13)
    # robots sit in front of the clutter and look into it (camera optical axis = robot +x), attitude within ~25 degrees
    robot[:, 0] = -3.0
    robot[:, 1:3] = (torch.rand(E, 2, generator=g) * 2 - 1) * 0.7
    e = (torch.rand(E, 3, generator=g) * 2 - 1) * 0.45
    cy, sy, cr, sr, cp, sp = torch.cos(e[:, 2] / 2), torch.sin(e[:, 2] / 2), torch.cos(e[:, 0] / 2), torch.sin(e[:, 0] / 2), torch.cos(e[:, 1] / 2), torch.sin(e[:, 1] / 2)
    robot[:, 3:7] = torch.stack([cy * sr * cp - sy * cr * sp, cy * cr * sp + sy * sr * cp, sy * cr * cp - cy * sr * sp, cy * cr * cp + sy * sr * sp], dim=1)
    mount = H.mounts(E, 1, seed=6)
    out["robot"], out["mount"] = robot.numpy(), mount.numpy()
    for name, (base, kw) in CASES.items():
        cfg = variant(base, **kw)
        pc = getattr(cfg, "return_pointcloud", False) or cfg.sensor_type.startswith("normal_faceID")
        shape = (E, 1, cfg.height, cfg.width, 3) if pc else (E, 1, cfg.height, cfg.width)
        gtd = {"robot_position": robot[:, 0:3].clone(), "robot_orientation": robot[:, 3:7].clone(), "gravity": torch.zeros(E, 3), "dt": 0.01,
               "robot_mass": torch.ones(E), "depth_range_pixels": torch.zeros(shape), "segmentation_pixels": torch.zeros((E, 1, cfg.height, cfg.width), dtype=torch.int32)}
        ws = WarpSensor(cfg, E, meshes, "cpu")
        ws.init_tensors(gtd)
        ws.sensor_local_position[:] = mount[..., 0:3]
        ws.sensor_local_orientation[:] = mount[..., 3:7]
        ws.update()  # pose composition -> the reference's kernels (through the stub) -> range limits -> normalisation
        out[f"{name}_pixels"] = gtd["depth_range_pixels"].numpy().copy()
        out[f"{name}_seg"] = gtd["segmentation_pixels"].numpy().copy()
        out[f"{name}_cfg"] = np.array([f"{k}={getattr(cfg, k)!r}" for k in FIELDS if hasattr(cfg, k)])
        s = ws.sensor
        if hasattr(s, "K_inv"):
            out[f"{name}_Kinv"], out[f"{name}_c"] = np.asarray(s.K_inv, np.float32), np.array([s.c_x, s.c_y])
        if hasattr(s, "ray_vectors"):
            out[f"{name}_ray_table"] = np.asarray(s.ray_vectors, np.float32)
        out[f"{name}_sensor_pos"], out[f"{name}_sensor_quat"] = ws.sensor_position.numpy().copy(), ws.sensor_orientation.numpy().copy()
        print(name, out[f"{name}_pixels"].shape, "pixels with a hit:", float((out[f"{name}_seg"] >= 0).mean()) if cfg.segmentation_camera or pc and cfg.sensor_type.startswith("normal") else "n/a")
    np.savez_compressed(os.path.join(HERE, "hp2_reference_sensors.npz"), **out)
    print("wrote hp2_reference_sensors.npz")


if __name__ == "__main__":
    main()
