"""Mesh and sphere geometry of environment assets, host side: OBJ / STL loading, the icosphere, the per-template BLAS, the
C ABI of the scene struct, and an EnvManager env with mesh assets on the CPU twin (oracle ray-caster)."""
import ctypes as C
import os
import struct

import numpy as np
import pytest
import torch

from aerial_gym_simulator_b200 import _lib, urdf
from aerial_gym_simulator_b200.hp2 import BLAS_LEAF_TRIS, build_blas, icosphere_triangles
from oracle import hp2_oracle as RO
from tests import _hp2_mesh_common as HM
from tests._cpu_stack import CpuRayScene, cpu_stack

QUAD_TRIS = np.array([[0, 0, 0, 1, 0, 0, 1, 1, 0], [0, 0, 0, 1, 1, 0, 0, 1, 0], [0, 0, 1, 1, 0, 1, 1, 1, 1]], np.float64)


def _write(path, text):
    with open(path, "w") as f:
        f.write(text)
    return path


def test_obj_and_stl_load_the_same_triangles(tmp_path):
    # OBJ: a quad (fan-triangulated) with v/vt/vn indices, then a triangle through negative indices
    obj = _write(tmp_path / "m.obj", "# test\nv 0 0 0\nv 1 0 0\nv 1 1 0\nv 0 1 0\nvt 0 0\nvn 0 0 1\n"
                                     "f 1/1/1 2/1/1 3//1 4\nv 0 0 1\nv 1 0 1\nv 1 1 1\nf -3 -2 -1\n")
    lines = ["solid m"]
    for t in QUAD_TRIS.reshape(-1, 3, 3):
        lines += ["facet normal 0 0 1", " outer loop"] + [f"  vertex {v[0]} {v[1]} {v[2]}" for v in t] + [" endloop", "endfacet"]
    ascii_stl = _write(tmp_path / "a.stl", "\n".join(lines + ["endsolid m"]) + "\n")
    with open(tmp_path / "b.stl", "wb") as f:
        f.write(b"solid-looking binary header".ljust(80, b" ") + struct.pack("<I", len(QUAD_TRIS)))
        for t in QUAD_TRIS:
            f.write(struct.pack("<3f", 0, 0, 1) + struct.pack("<9f", *t) + b"\0\0")
    for p in (obj, ascii_stl, tmp_path / "b.stl"):
        assert np.array_equal(urdf.load_mesh(str(p)), QUAD_TRIS), p
    scaled = urdf.load_mesh(str(obj), (2.0, 3.0, 0.5))
    assert np.array_equal(scaled.reshape(-1, 3), QUAD_TRIS.reshape(-1, 3) * [2.0, 3.0, 0.5])


def test_unsupported_mesh_inputs_raise(tmp_path):
    dae = _write(tmp_path / "m.dae", "<COLLADA/>")
    with pytest.raises(ValueError, match="m.dae"):
        urdf.load_mesh(str(dae))
    with pytest.raises(ValueError, match="package://pkg/m.obj"):
        urdf.load_mesh("package://pkg/m.obj")
    _write(tmp_path / "a.urdf", HM.URDF_MESH.format(name="a", mesh="m.dae", scale="1 1 1"))
    with pytest.raises(ValueError, match="m.dae"):
        urdf.visual_parts(urdf.parse_urdf(str(tmp_path / "a.urdf")))


def test_icosphere():
    t = icosphere_triangles(0.37)
    assert t.shape == (1280, 9)
    v = t.reshape(-1, 3)
    assert len(np.unique(v, axis=0)) == 642
    assert np.allclose(np.linalg.norm(v.astype(np.float64), axis=1), 0.37, rtol=1e-6)


@pytest.mark.parametrize("n_sub,seed", [(0, 1), (2, 2), (3, 3)])
def test_blas_invariants(n_sub, seed):
    tris = HM.bumpy_mesh(seed, n_sub)[: 20 * 4 ** n_sub - seed]  # odd counts too
    b = build_blas(tris)
    topo, levels, order = b["topo"], b["levels"], b["order"]
    assert sorted(order.tolist()) == list(range(len(tris)))
    v = tris[order].reshape(-1, 3, 3)
    covered = np.zeros(len(tris), int)
    box = {}

    def visit(i, depth):
        assert depth < _lib.BLAS_MAX_DEPTH and levels[depth] <= i < levels[depth + 1]
        a, n = topo[i]
        if n > 0:
            assert n <= BLAS_LEAF_TRIS
            covered[a:a + n] += 1
            p = v[a:a + n].reshape(-1, 3)
        else:
            p = np.concatenate([visit(a, depth + 1), visit(a + 1, depth + 1)])
        box[i] = (p.min(0), p.max(0))
        return p

    visit(0, 0)
    assert (covered == 1).all() and len(box) == len(topo)
    for i, (a, n) in enumerate(topo):
        if n == 0:
            for c in (a, a + 1):
                assert (box[i][0] <= box[c][0]).all() and (box[c][1] <= box[i][1]).all()
    b2 = build_blas(tris.copy())
    assert all(np.array_equal(b[k], b2[k]) for k in b)


def test_shipped_environment_assets_are_boxes_and_cylinders():
    from aerial_gym_simulator_b200.config.asset_config import _ENV_ASSETS
    n = 0
    for root, _, files in os.walk(_ENV_ASSETS):
        for f in files:
            if f.endswith(".urdf"):
                parts = urdf.visual_parts(urdf.parse_urdf(os.path.join(root, f)))
                assert all(obb is not None and len(t) <= 12 for _, _, t, obb in parts), f
                n += 1
    assert n > 10


def test_scene_struct_abi():
    assert _lib.load().agx_sizeof(3) == C.sizeof(_lib.AgxHp2Scene)
    assert _lib.AgxHp2Scene.obb.offset < _lib.AgxHp2Scene.num_meshes.offset  # new fields appended


class CpuMeshRayScene(CpuRayScene):
    """CPU twin of a RayScene with mesh templates: the oracle sees them as templates of their full size, in file order"""

    def __init__(self, templates, tmpl_seg_base, tmpl_seg_mask, obj_template, obj_seg_counter, obj_pose, device="cpu",
                 tris_per_object=None, bounds_min=None, bounds_max=None, tmpl_obb=None, mesh_templates=None):
        self.mesh_templates = list(mesh_templates or [])
        super().__init__(list(templates) + self.mesh_templates, tmpl_seg_base, tmpl_seg_mask, obj_template, obj_seg_counter,
                         obj_pose, device, None, bounds_min, bounds_max, tmpl_obb)


def test_env_manager_with_mesh_assets_on_cpu_twin(tmp_path):
    import aerial_gym_simulator_b200.env_manager.env_manager as EM
    from aerial_gym_simulator_b200.registry._core import env_config_registry
    from aerial_gym_simulator_b200.sim import SimBuilder

    folder = HM.write_mesh_assets(str(tmp_path / "assets"))
    env_config_registry.register("mesh_test_env_cpu", HM.mesh_env_cfg(folder))
    N = 3
    with cpu_stack():
        EM.RayScene = CpuMeshRayScene
        env = SimBuilder().build_env("base_sim", "mesh_test_env_cpu", "base_quadrotor_with_camera", "lee_velocity_control", "cpu",
                                     args={"seed": 5}, num_envs=N, use_warp=True, headless=True)
        sc = env.scene
        assert isinstance(sc, CpuMeshRayScene) and len(sc.mesh_templates) == 2
        assert {len(m) for m in sc.mesh_templates} == {320, 1280}
        env.reset()
        gtd = env.get_obs()
        ast = gtd["env_asset_state_tensor"]
        ast[:, :, 0:3] = gtd["robot_position"][:, None, :] + torch.tensor([1.2, 0.0, 0.0])  # in front of the camera
        ast[:, 0, 0:3] = gtd["robot_position"] + torch.tensor([0.0, 0.0, 0.5])  # and one close to the robot
        for _ in range(2):  # the obstacle step re-poses the scene (a refit of every mesh object)
            env.step(actions=torch.zeros(N, 4), env_actions=torch.zeros(N, 4, 6))
        env.render()
        # independent restatement: URDF -> triangles -> oracle world mesh, posed by the gathered asset rows, faces in file order
        parts = {f: urdf.visual_parts(urdf.parse_urdf(os.path.join(folder, f)))[0][2] for f in ("ball.urdf", "rock.urdf")}
        assert sorted(len(t) for t in parts.values()) == [320, 1280]
        order = [next(t for t in parts.values() if np.array_equal(t, m)) for m in sc.mesh_templates]
        offs = np.concatenate([[0], np.cumsum([len(t) for t in order])]).astype(np.int32)
        tt = np.concatenate(order)
        ones = np.ones(len(tt), np.int32)
        tris, segs, cnt = RO.build_world_tris(env._obj_pose.numpy(), sc.obj_template.numpy(), sc.obj_seg_counter.numpy(), offs, tt,
                                              0 * ones, ones, sc.K * 1280)
        assert np.array_equal(tris[:, :cnt.max()], sc._tris[:, :cnt.max()]) and (cnt == sc._cnt).all()
        so, _ = HM.H.oracle_sensor(env.sensor_cfg, fuse=not env.sensor.noise_enabled)
        so.segmentation = int(env.sensor.seg_pixels is not None)
        root = env.engine.root_state[:, :7].numpy()
        ref, ref_seg = RO.cast(so, root, env.sensor_mount.numpy(), None, tris, segs, cnt)
        assert np.array_equal(gtd["depth_range_pixels"].numpy(), ref)
        if ref_seg is not None:
            assert np.array_equal(gtd["segmentation_pixels"].numpy(), ref_seg)
        assert (ref_seg >= 100).mean() > 0.2 if ref_seg is not None else (ref < 1.0).mean() > 0.2  # the mesh obstacles are seen
        env.collision_tensor.zero_()
        env.compute_observations()
        flags, _ = RO.collide(root, float(env.robot.collision_radius), tris, cnt)
        assert np.array_equal(env.collision_tensor.bool().numpy(), flags)
