"""Ray-caster with mesh objects: one fixed workload, one JSON line.

Workload: 2048 envs, one 64x48 depth + segmentation camera per env (BaseDepthCameraConfig values), a scene of 6 walls (boxes,
triangle clusters) + 20 mesh obstacles (14 of 1280 and 6 of 5120 triangles: seeded bumpy icospheres) + 4 spheres (URDF <sphere>:
1280-triangle icospheres) per env, every object randomly posed inside the walls.
Reported: cast rays/s, agx_hp2_update_scene time of a full reset (transform + BLAS refit + top-level build), agx_hp2_collide time,
the same scene with every mesh / sphere replaced by its bounding box through the cluster path, and the brute-force oracle on a few
envs as the CPU baseline (kind "port": the project's own C restatement, not the reference).

python tools/hp2_mesh_bench.py [--envs 2048] [--iters 50] [--out FILE]"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from aerial_gym_simulator_b200.hp2 import RayScene, RaySensor, box_obb, box_triangles, icosphere_triangles  # noqa: E402
from oracle import hp2_oracle as RO  # noqa: E402


class Cam:
    sensor_type, num_sensors, height, width = "camera", 1, 48, 64
    horizontal_fov_deg, max_range, min_range = 87.0, 10.0, 0.2
    calculate_depth, return_pointcloud, pointcloud_in_world_frame = True, False, False
    segmentation_camera, normalize_range = True, True
    far_out_of_range_value, near_out_of_range_value = 10.0, -10.0
    euler_frame_rot_deg = [-90.0, 0, -90.0]

    class sensor_noise:
        enable_sensor_noise = False


def bumpy(seed, n_sub):
    t = icosphere_triangles(1.0, n_sub).reshape(-1, 3).astype(np.float64)
    keys, inv = np.unique(t, axis=0, return_inverse=True)
    r = 0.5 * (1.0 + 0.4 * np.random.default_rng(seed).random(len(keys)))
    return (t * r[inv.reshape(-1)][:, None]).astype(np.float32).reshape(-1, 9)


def workload(E, seed=0):
    walls = [(12.0, 0.2, 6.0, (0, 6, 0)), (12.0, 0.2, 6.0, (0, -6, 0)), (0.2, 12.0, 6.0, (6, 0, 0)), (0.2, 12.0, 6.0, (-6, 0, 0)),
             (12.0, 12.0, 0.2, (0, 0, -3)), (12.0, 12.0, 0.2, (0, 0, 3))]
    meshes = [bumpy(i, 3) for i in range(14)] + [bumpy(100 + i, 4) for i in range(6)] + [icosphere_triangles(0.4)] * 4
    g = torch.Generator().manual_seed(seed)
    K = len(walls) + len(meshes)
    pose = torch.zeros(E, K, 13)
    pose[..., 6] = 1.0
    for k, (_, _, _, p) in enumerate(walls):
        pose[:, k, 0:3] = torch.tensor(p, dtype=torch.float32)
    pose[:, 6:, 0:3] = (torch.rand(E, K - 6, 3, generator=g) * 2 - 1) * torch.tensor([5.0, 5.0, 2.5])
    q = torch.randn(E, K - 6, 4, generator=g)
    pose[:, 6:, 3:7] = q / q.norm(dim=-1, keepdim=True)
    tm = np.tile(np.arange(K, dtype=np.int32), (E, 1))
    ctr = (100 + np.arange(E * K, dtype=np.int32)).reshape(E, K)
    robot = torch.zeros(E, 13)
    robot[:, 0:3] = (torch.rand(E, 3, generator=g) * 2 - 1) * torch.tensor([4.0, 4.0, 2.0])
    yaw = torch.rand(E, generator=g) * 2 * math.pi
    robot[:, 5], robot[:, 6] = torch.sin(yaw / 2), torch.cos(yaw / 2)
    return [box_triangles(w[:3]) for w in walls], [box_obb(w[:3]) for w in walls], meshes, tm, ctr, pose, robot


def timed(fn, iters):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters  # ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=2048)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--oracle-envs", type=int, default=4)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("hp2_mesh_bench needs a CUDA device")
    dev = "cuda:0"
    E = a.envs
    walls, wall_obbs, meshes, tm, ctr, pose, robot = workload(E)
    T, M = len(walls), len(meshes)
    n_mesh_tris = sum(len(m) for m in meshes)
    pose_d, robot_d = pose.to(dev), robot.to(dev)
    res = {"workload": dict(envs=E, image="64x48 depth+seg", walls_as_boxes=T, mesh_obstacles=20, mesh_tris=[1280] * 14 + [5120] * 6,
                            spheres=4, sphere_tris=1280, tris_per_env=T * 12 + n_mesh_tris)}
    # mesh path
    scene = RayScene(walls, [0] * (T + M), [1] * (T + M), tm, ctr, pose_d, dev,
                     tmpl_obb=np.concatenate([np.stack(wall_obbs), np.zeros((M, 16), np.float32)]), mesh_templates=meshes)
    pix = torch.zeros(E, 1, 48, 64, device=dev)
    seg = torch.zeros(E, 1, 48, 64, dtype=torch.int32, device=dev)
    sensor = RaySensor(Cam, scene, robot_d, pix, seg)
    scene.update()
    rays = E * 48 * 64
    t_cast = timed(sensor.capture, a.iters)
    t_upd = timed(scene.update, max(5, a.iters // 5))
    crashes = torch.zeros(E, dtype=torch.bool, device=dev)
    t_col = timed(lambda: scene.collide(robot_d, 0.18384776, crashes), a.iters)
    res["mesh"] = dict(cast_ms=t_cast, cast_rays_per_s=rays / (t_cast * 1e-3), update_scene_full_reset_ms=t_upd, collide_us=t_col * 1e3,
                       bytes_mesh_storage_per_env=int(scene.c.mesh_tris_per_env) * 48 + int(scene.c.mesh_nodes_per_env) * 32)
    hit_frac = float((seg >= 0).float().mean())
    res["mesh"]["hit_fraction"] = hit_frac
    # oracle (CPU baseline) on a sample of envs, checked against the GPU image
    sub = list(range(a.oracle_envs))
    allt = walls + meshes
    offs = np.concatenate([[0], np.cumsum([len(t) for t in allt])]).astype(np.int32)
    tt = np.concatenate(allt)
    z, o = np.zeros(len(tt), np.int32), np.ones(len(tt), np.int32)
    tris, segs, cnt = RO.build_world_tris(pose[sub, :, :7].numpy(), tm[sub], ctr[sub], offs, tt, z, o, T * 12 + n_mesh_tris)
    so = RO.Hp2oSensor()
    so.kind, so.width, so.height, so.num_sensors, so.calculate_depth, so.segmentation = 0, 64, 48, 1, 1, 1
    so.fuse_epilogue, so.normalize_range = 1, 1
    kinv, cx, cy = RO.camera_kinv(64, 48, 87.0)
    for i, v in enumerate(kinv.reshape(-1)):
        so.kinv[i] = float(v)
    so.c_x, so.c_y = cx, cy
    so.far_plane = so.max_range = 10.0
    so.min_range, so.far_out_of_range_value, so.near_out_of_range_value = 0.2, 10.0, -10.0
    for i, v in enumerate(RO.quat_from_euler_deg([-90.0, 0, -90.0])):
        so.frame_quat[i] = float(v)
    m = np.tile(np.array([0, 0, 0, 0, 0, 0, 1], np.float32), (len(sub), 1, 1))
    t0 = time.perf_counter()
    ref_pix, ref_seg = RO.cast(so, robot[sub, :7].numpy(), m, None, tris, segs, cnt)
    t_or = time.perf_counter() - t0
    res["cpu_baseline"] = dict(kind="port", envs=len(sub), rays_per_s=len(sub) * 48 * 64 / t_or,
                               bit_identical=bool(np.array_equal(pix[sub].cpu().numpy(), ref_pix) and np.array_equal(seg[sub].cpu().numpy(), ref_seg)))
    del scene, sensor
    torch.cuda.empty_cache()
    # the same scene with every mesh / sphere as its bounding box (cluster path)
    boxes, obbs = [], []
    for mt in meshes:
        v = mt.reshape(-1, 3)
        lo, hi = v.min(0), v.max(0)
        boxes.append((box_triangles(hi - lo).reshape(-1, 3) + (lo + hi) / 2).reshape(-1, 9).astype(np.float32))
        obbs.append(box_obb(hi - lo, None, (lo + hi) / 2))
    scene_b = RayScene(walls + boxes, [0] * (T + M), [1] * (T + M), tm, ctr, pose_d, dev, tmpl_obb=np.stack(wall_obbs + obbs))
    sensor_b = RaySensor(Cam, scene_b, robot_d, pix, seg)
    scene_b.update()
    t_cast_b = timed(sensor_b.capture, a.iters)
    t_upd_b = timed(scene_b.update, max(5, a.iters // 5))
    t_col_b = timed(lambda: scene_b.collide(robot_d, 0.18384776, crashes), a.iters)
    res["boxes_instead"] = dict(cast_ms=t_cast_b, cast_rays_per_s=rays / (t_cast_b * 1e-3), update_scene_full_reset_ms=t_upd_b,
                                collide_us=t_col_b * 1e3)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    res["gpu"] = dict(name=torch.cuda.get_device_name(0), nvidia_smi=smi.stdout.strip().splitlines()[0] if smi.returncode == 0 else None)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
