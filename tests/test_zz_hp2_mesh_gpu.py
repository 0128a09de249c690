"""Mesh objects (URDF <mesh> / <sphere> visuals) in the CUDA ray-caster and collision test: bit-identical to the brute-force
oracle on mixed box + mesh + sphere scenes -- pixels, segmentation ids, face ids, collision flags and min distances."""
import os

import numpy as np
import pytest
import torch

from aerial_gym_simulator_b200 import urdf
from aerial_gym_simulator_b200.hp2 import RayScene, RaySensor
from oracle import hp2_oracle as RO
from tests import _hp2_common as H
from tests import _hp2_mesh_common as HM

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(autouse=True)
def _needs_the_kernels():
    if DEV == "cpu":  # the CPU dry run of the GPU test text: these tests check the mesh kernels themselves, which have no CPU twin
        pytest.skip("the mesh kernels have no CPU twin")


def build(sc, cfg, seed, mount_seed=None):
    t, b, m = HM.scene_templates(sc)
    scene = RayScene(t, b, m, sc["tm"], sc["ctr"], sc["pose"].to(DEV), DEV, tmpl_obb=sc["obbs"], mesh_templates=sc["meshes"])
    scene.update()
    E = sc["E"]
    robot = H.robot_poses(E, seed)
    mount = H.mounts(E, 1, mount_seed) if mount_seed is not None else None
    pc = cfg.return_pointcloud or cfg.sensor_type.startswith("normal_faceID")
    pix = torch.zeros((E, 1, cfg.height, cfg.width, 3) if pc else (E, 1, cfg.height, cfg.width), device=DEV)
    seg = torch.zeros(E, 1, cfg.height, cfg.width, dtype=torch.int32, device=DEV) if cfg.segmentation_camera else None
    sensor = RaySensor(cfg, scene, robot.to(DEV), pix, seg, mount.to(DEV) if mount is not None else None)
    return scene, sensor, robot, mount


def oracle_cast(sc, cfg, sensor, robot, mount):
    tris, segs, cnt = HM.oracle_tris(sc)
    so, table = H.oracle_sensor(cfg, fuse=not sensor.noise_enabled)
    if sensor.ray_table is not None:
        table = sensor.ray_table.cpu().numpy()
    m = mount.numpy() if mount is not None else np.tile(np.array([0, 0, 0, 0, 0, 0, 1], np.float32), (sc["E"], 1, 1))
    return RO.cast(so, robot[:, :7].numpy(), m, table, tris, segs, cnt)


def check(sensor, ref_pix, ref_seg):
    torch.cuda.synchronize()
    got = sensor.pixels.cpu().numpy()
    assert np.array_equal(got, ref_pix), f"{(got != ref_pix).sum()} / {got.size} pixels differ"
    if ref_seg is not None:
        assert np.array_equal(sensor.seg_pixels.cpu().numpy(), ref_seg)


SENSORS = {
    "depth_seg": (H.CamCfg, dict()),
    "range_seg": (H.CamCfg, dict(calculate_depth=False)),
    "pointcloud_sensor_frame": (H.CamCfg, dict(return_pointcloud=True)),
    "pointcloud_world": (H.CamCfg, dict(return_pointcloud=True, pointcloud_in_world_frame=True, normalize_range=False)),
    "lidar": (H.LidarCfg, dict()),
    "stereo": (H.CamCfg, dict(sensor_type="stereo_camera", baseline=-0.095, height=40, width=56)),
    "normal_faceid_camera": (H.CamCfg, dict(sensor_type="normal_faceID_camera", return_pointcloud=True, normal_in_world_frame=True,
                                            pointcloud_in_world_frame=True, height=24, width=40)),
    "normal_faceid_lidar": (H.LidarCfg, dict(sensor_type="normal_faceID_lidar", return_pointcloud=True, normal_in_world_frame=False,
                                             pointcloud_in_world_frame=False, height=16, width=48)),
}


@pytest.mark.parametrize("name", list(SENSORS))
def test_sensors_match_oracle_on_mixed_scenes(name):
    base, kw = SENSORS[name]
    cfg = H.cfg_variant(base, **kw)
    sc = HM.make_mixed_scene(5, 24, seed=11, extent=3.0, parked=4)
    scene, sensor, robot, mount = build(sc, cfg, seed=2, mount_seed=3)
    sensor.capture()
    ref_pix, ref_seg = oracle_cast(sc, cfg, sensor, robot, mount)
    check(sensor, ref_pix, ref_seg)
    if "faceid" in name:
        assert (ref_seg > 24 * 12).any()  # faces beyond any box cluster: mesh triangles were hit
    elif ref_seg is not None:
        assert (ref_seg >= 100).mean() > 0.05


def test_masked_update_changes_only_masked_envs():
    cfg = H.cfg_variant(H.CamCfg, height=16, width=24)
    sc = HM.make_mixed_scene(4, 10, seed=60, extent=3.0)
    scene, sensor, robot, mount = build(sc, cfg, seed=9)
    sensor.capture()
    before = sensor.pixels.clone()
    g = torch.Generator().manual_seed(1)
    new_pose = sc["pose"].clone()
    new_pose[..., 0:3] = (torch.rand(4, 10, 3, generator=g) * 2 - 1) * 3
    scene.obj_pose.copy_(new_pose.to(DEV))
    scene.update(torch.tensor([True, False, True, False], device=DEV))
    sensor.capture()
    torch.cuda.synchronize()
    assert torch.equal(sensor.pixels[1], before[1]) and torch.equal(sensor.pixels[3], before[3])
    mixed = sc["pose"].clone()
    mixed[0], mixed[2] = new_pose[0], new_pose[2]
    check(sensor, *oracle_cast(dict(sc, pose=mixed), cfg, sensor, robot, mount))


def test_scene_too_large_for_shared_memory():
    """400 objects x 12 cluster slots = 230 KB of slabs per env: the top level is read through L2 as well"""
    sc = HM.make_mixed_scene(2, 400, seed=50, extent=6.0)
    for cfg in (H.cfg_variant(H.CamCfg, height=12, width=16), H.cfg_variant(H.LidarCfg, height=8, width=64)):
        scene, sensor, robot, mount = build(sc, cfg, seed=8)
        sensor.capture()
        check(sensor, *oracle_cast(sc, cfg, sensor, robot, mount))


def test_collision_flags_and_min_dist_match_oracle():
    E = 512
    sc = HM.make_mixed_scene(E, 12, seed=100, extent=2.0, parked=3)
    t, b, m = HM.scene_templates(sc)
    scene = RayScene(t, b, m, sc["tm"], sc["ctr"], sc["pose"].to(DEV), DEV, mesh_templates=sc["meshes"])
    scene.update()
    robot = H.robot_poses(E, 12, extent=2.0)
    crashes = torch.zeros(E, dtype=torch.bool, device=DEV)
    md = torch.zeros(E, device=DEV)
    scene.collide(robot.to(DEV), 0.18384776, crashes, md)
    tris, segs, cnt = HM.oracle_tris(sc)
    ref_hit, ref_d2 = RO.collide(robot[:, :7].numpy(), 0.18384776, tris, cnt)
    torch.cuda.synchronize()
    assert np.array_equal(crashes.cpu().numpy(), ref_hit)
    assert np.array_equal(md.cpu().numpy(), np.sqrt(ref_d2))
    assert 0 < ref_hit.sum() < E
    c2 = torch.zeros(E, dtype=torch.bool, device=DEV)
    scene.collide(robot.to(DEV), 0.18384776, c2, None)
    assert torch.equal(c2, crashes)


def test_boxes_as_one_obj_render_like_box_visuals(tmp_path):
    g = np.random.default_rng(7)
    sizes, xyz = g.random((20, 3)) * 0.8 + 0.2, (g.random((20, 3)) * 2 - 1) * 3
    num = lambda v: " ".join(repr(float(x)) for x in v)
    vis = "".join(f'    <visual><origin xyz="{num(p)}"/><geometry><box size="{num(s)}"/></geometry></visual>\n' for s, p in zip(sizes, xyz))
    with open(tmp_path / "boxes.urdf", "w") as f:
        f.write(HM.URDF_BOXES.format(visuals=vis))
    box_parts = urdf.visual_parts(urdf.parse_urdf(str(tmp_path / "boxes.urdf")))
    assert len(box_parts) == 20
    HM.write_obj(tmp_path / "boxes.obj", np.concatenate([t for _, _, t, _ in box_parts]))
    with open(tmp_path / "mesh.urdf", "w") as f:
        f.write(HM.URDF_MESH.format(name="m", mesh="boxes.obj", scale="1 1 1"))
    (_, _, mesh, obb), = urdf.visual_parts(urdf.parse_urdf(str(tmp_path / "mesh.urdf")))
    assert obb is None and np.array_equal(mesh, np.concatenate([t for _, _, t, _ in box_parts]))
    E = 4
    pose = torch.zeros(E, 20, 13)
    pose[..., 6] = 1.0
    cfg = H.cfg_variant(H.CamCfg, height=48, width=64)
    robot = H.robot_poses(E, 3, extent=0.5).to(DEV)
    outs = []
    for mesh_scene in (False, True):
        if mesh_scene:
            p = pose[:, :1].contiguous().to(DEV)
            scene = RayScene([], [0], [1], np.zeros((E, 1), np.int32), np.zeros((E, 1), np.int32), p, DEV, mesh_templates=[mesh])
        else:
            scene = RayScene([t for _, _, t, _ in box_parts], [0] * 20, [1] * 20, np.tile(np.arange(20, dtype=np.int32), (E, 1)),
                             np.zeros((E, 20), np.int32), pose.to(DEV), DEV, tmpl_obb=np.stack([o for *_, o in box_parts]))
        scene.update()
        pix = torch.zeros(E, 1, 48, 64, device=DEV)
        RaySensor(cfg, scene, robot, pix, None).capture()
        outs.append(pix.cpu())
    assert (outs[0] < 1.0).any() and torch.equal(outs[0], outs[1])


def test_sim_builder_env_with_mesh_assets_and_env_actions(tmp_path):
    from aerial_gym_simulator_b200.registry._core import env_config_registry
    from aerial_gym_simulator_b200.sim import SimBuilder

    folder = HM.write_mesh_assets(str(tmp_path / "assets"))
    env_config_registry.register("mesh_test_env_gpu", HM.mesh_env_cfg(folder))
    N = 8
    env = SimBuilder().build_env("base_sim", "mesh_test_env_gpu", "base_quadrotor_with_camera", "lee_velocity_control", DEV,
                                 args={"seed": 5}, num_envs=N, use_warp=True, headless=True)
    sc = env.scene
    assert sc.c.num_meshes == 2
    env.reset()
    gtd = env.get_obs()
    ast = gtd["env_asset_state_tensor"]
    ast[:, :, 0:3] = gtd["robot_position"][:, None, :] + torch.tensor([1.2, 0.0, 0.0], device=DEV)
    twist = torch.zeros(N, 4, 6, device=DEV)
    twist[..., 1], twist[..., 5] = 0.5, 0.8  # a dynamic re-pose through env_actions: every mesh object is refit
    for _ in range(2):
        env.step(actions=torch.zeros(N, 4, device=DEV), env_actions=twist)
    env.render()
    torch.cuda.synchronize()
    meshes = [sc.mesh_tris.cpu().numpy()[a:b][np.argsort(sc.mesh_tri_index.cpu().numpy()[a:b])]
              for a, b in zip(sc.mesh_tri_offset.cpu().numpy()[:-1], sc.mesh_tri_offset.cpu().numpy()[1:])]
    T = int(sc.c.num_templates) - 2
    seg_b = sc.mesh_seg.cpu().numpy()
    allt = meshes
    offs = np.concatenate([[0], np.cumsum([len(t) for t in allt])]).astype(np.int32)
    tt = np.concatenate(allt)
    sb = np.concatenate([np.full(len(t), seg_b[i, 0], np.int32) for i, t in enumerate(allt)])
    sm = np.concatenate([np.full(len(t), seg_b[i, 1], np.int32) for i, t in enumerate(allt)])
    tris, segs, cnt = RO.build_world_tris(env._obj_pose.cpu().numpy(), sc.obj_template.cpu().numpy() - T, sc.obj_seg_counter.cpu().numpy(),
                                          offs, tt, sb, sm, sc.K * 1280)
    so, _ = H.oracle_sensor(env.sensor_cfg, fuse=not env.sensor.noise_enabled)
    so.segmentation = int(env.sensor.seg_pixels is not None)
    root = env.engine.root_state[:, :7].cpu().numpy()
    ref, ref_seg = RO.cast(so, root, env.sensor_mount.cpu().numpy(), None, tris, segs, cnt)
    assert np.array_equal(gtd["depth_range_pixels"].cpu().numpy(), ref)
    if ref_seg is not None:
        assert np.array_equal(gtd["segmentation_pixels"].cpu().numpy(), ref_seg)
    assert (ref < 1.0).mean() > 0.05
    crashes = torch.zeros(N, dtype=torch.bool, device=DEV)
    sc.collide(env.engine.root_state, float(env.robot.collision_radius), crashes)
    flags, _ = RO.collide(root, float(env.robot.collision_radius), tris, cnt)
    assert np.array_equal(crashes.cpu().numpy(), flags)
