"""HP2 throughput on the BASELINE.json sensor configs (synthetic randomly posed box scenes).
Prints one JSON line per config.  Run on an H100: python tools/hp2_sweep.py [--quick]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from aerial_gym_simulator_b200.hp2 import RayScene, RaySensor, box_obb, box_triangles  # noqa: E402


def cam_cfg(h, w):
    class C:
        sensor_type, num_sensors, height, width = "camera", 1, h, w
        horizontal_fov_deg, max_range, min_range = 87.0, 10.0, 0.2
        calculate_depth, return_pointcloud, pointcloud_in_world_frame = True, False, False
        segmentation_camera, normalize_range = True, True
        far_out_of_range_value, near_out_of_range_value = 10.0, -10.0
        euler_frame_rot_deg = [-90.0, 0, -90.0]
    return C


def lidar_cfg(h, w):
    class C:
        sensor_type, num_sensors, height, width = "lidar", 1, h, w
        horizontal_fov_deg_min, horizontal_fov_deg_max, vertical_fov_deg_min, vertical_fov_deg_max = -180, 180, 0, 90
        max_range, min_range = 20.0, 0.5
        return_pointcloud, pointcloud_in_world_frame, segmentation_camera, normalize_range = False, False, True, True
        far_out_of_range_value, near_out_of_range_value = 10.0, -10.0
        euler_frame_rot_deg = [0.0, 0.0, 0.0]
    return C


def run(name, E, K, cfg, frames, extent, dev="cuda:0"):
    g = torch.Generator().manual_seed(3)
    sizes = torch.rand(5, 3, generator=g) * 1.2 + 0.15
    templates = [box_triangles(s.tolist()) for s in sizes]
    pose = torch.zeros(E, K, 13)
    pose[..., 0:3] = (torch.rand(E, K, 3, generator=g) * 2 - 1) * extent
    q = torch.randn(E, K, 4, generator=g)
    pose[..., 3:7] = q / q.norm(dim=-1, keepdim=True)
    tm = torch.randint(0, 5, (E, K), generator=g).numpy()
    ctr = (100 + torch.arange(E * K).reshape(E, K) % 100000).numpy()
    scene = RayScene(templates, [0] * 5, [1] * 5, tm, ctr, pose.to(dev), dev, tmpl_obb=np.stack([box_obb(s.tolist()) for s in sizes]))
    robot = torch.zeros(E, 13)
    robot[:, 0:3] = (torch.rand(E, 3, generator=g) * 2 - 1) * (extent * 0.8)
    rq = torch.randn(E, 4, generator=g)
    robot[:, 3:7] = rq / rq.norm(dim=-1, keepdim=True)
    H, W = cfg.height, cfg.width
    pix = torch.zeros(E, 1, H, W, device=dev)
    seg = torch.zeros(E, 1, H, W, dtype=torch.int32, device=dev)
    sensor = RaySensor(cfg, scene, robot.to(dev), pix, seg)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); scene.update(); e1.record(); torch.cuda.synchronize()
    upd = e0.elapsed_time(e1)
    for _ in range(2):
        sensor.capture()
    torch.cuda.synchronize()
    e0.record()
    for _ in range(frames):
        sensor.capture()
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / frames
    rays = E * H * W
    print(json.dumps({"config": name, "envs": E, "objects_per_env": K, "triangles_per_env": K * 12, "image": [H, W],
                      "rays_per_frame": rays, "ms_per_frame": ms, "rays_per_s": rays / ms * 1e3,
                      "hit_fraction": float((seg >= 0).float().mean()), "scene_update_ms": upd,
                      "scene_in_shared_memory": K * 12 * 48 + 4096 < 200000}))


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true")
    a = ap.parse_args()
    f = 3 if a.quick else 10
    run("north-star depth 64x48, 8192 envs, 44 boxes", 8192, 44, cam_cfg(48, 64), f * 3, 5.0)
    run("depth 135x240 (shipped camera), 1024 envs, 44 boxes", 1024, 44, cam_cfg(135, 240), f, 5.0)
    run("BASELINE cfg#3 depth 270x480, 8192 envs, 1024 boxes", 8192 if not a.quick else 1024, 1024, cam_cfg(270, 480), max(1, f // 5), 8.0)
    run("BASELINE cfg#4 LiDAR 64x512 + seg, 16384 envs, 44 boxes", 16384 if not a.quick else 2048, 44, lidar_cfg(64, 512), f, 6.0)
