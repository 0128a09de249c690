"""Scene and asset builders for the mesh-object HP2 tests (boxes + OBJ meshes + spheres), oracle side in numpy."""
import os

import numpy as np
import torch

from aerial_gym_simulator_b200.hp2 import icosphere_triangles
from oracle import hp2_oracle as RO

from . import _hp2_common as H


def bumpy_mesh(seed, n_sub=3, radius=0.6):
    """an irregular closed mesh (icosphere with seeded radial bumps): 20 * 4^n_sub triangles"""
    t = icosphere_triangles(1.0, n_sub).reshape(-1, 3).astype(np.float64)
    g = np.random.default_rng(seed)
    keys, inv = np.unique(t, axis=0, return_inverse=True)
    r = radius * (1.0 + 0.35 * g.random(len(keys)))
    return (t * r[inv.reshape(-1)][:, None]).astype(np.float32).reshape(-1, 9)


def write_obj(path, tris):
    """one vertex per corner, float32 values written with enough digits to round-trip"""
    with open(path, "w") as f:
        for v in np.asarray(tris, np.float32).reshape(-1, 3):
            f.write("v %s %s %s\n" % tuple(repr(float(x)) for x in v))
        for i in range(len(tris)):
            f.write(f"f {3 * i + 1} {3 * i + 2} {3 * i + 3}\n")


def make_mixed_scene(E, K, seed, extent=4.0, parked=0, n_meshes=2, sphere_radius=0.5):
    """K objects per env drawn from 5 box templates, `n_meshes` bumpy meshes and one icosphere (mesh templates)."""
    sc = H.make_scene(E, K, seed, extent=extent, parked=parked)
    meshes = [bumpy_mesh(seed + i, n_sub=3 if i % 2 == 0 else 2) for i in range(n_meshes)] + [icosphere_triangles(sphere_radius)]
    g = torch.Generator().manual_seed(seed + 1000)
    T = len(sc["templates"])
    tm = torch.randint(0, T + len(meshes), (E, K), generator=g).numpy().astype(np.int32)
    tm[:, 0] = T  # every env has at least one mesh object, first in the concatenated mesh
    sc.update(tm=tm, meshes=meshes, obbs=np.concatenate([sc["obbs"], np.zeros((len(meshes), 16), np.float32)]))
    return sc


def scene_templates(sc):
    """(templates, seg_base, seg_mask) arguments of RayScene for a make_mixed_scene / make_scene dict"""
    n = len(sc["templates"]) + len(sc.get("meshes", []))
    return sc["templates"], [0] * n, [1] * n


def oracle_tris(sc):
    """world triangles of the env's concatenated mesh, templates and meshes in file order"""
    allt = list(sc["templates"]) + list(sc.get("meshes", []))
    offs = np.zeros(len(allt) + 1, np.int32)
    offs[1:] = np.cumsum([len(t) for t in allt])
    tris = np.concatenate(allt)
    max_tris = sc["K"] * max(len(t) for t in allt)
    return RO.build_world_tris(sc["pose"][..., :7].numpy(), sc["tm"], sc["ctr"], offs, tris, np.zeros(len(tris), np.int32),
                               np.ones(len(tris), np.int32), max_tris)


URDF_MESH = """<?xml version="1.0"?>
<robot name="{name}">
  <link name="base_link">
    <visual><origin xyz="0 0 0" rpy="0 0 0"/><geometry><mesh filename="{mesh}" scale="{scale}"/></geometry></visual>
  </link>
</robot>
"""
URDF_SPHERE = """<?xml version="1.0"?>
<robot name="ball">
  <link name="base_link">
    <visual><origin xyz="0.1 0 0" rpy="0 0 0"/><geometry><sphere radius="{r}"/></geometry></visual>
  </link>
</robot>
"""
URDF_BOXES = """<?xml version="1.0"?>
<robot name="boxes">
  <link name="base_link">
{visuals}  </link>
</robot>
"""


def write_mesh_assets(folder, seed=0):
    """an asset folder with one OBJ-mesh obstacle and one sphere obstacle (URDFs + mesh file)"""
    os.makedirs(folder, exist_ok=True)
    write_obj(os.path.join(folder, "rock.obj"), bumpy_mesh(seed, n_sub=2))
    with open(os.path.join(folder, "rock.urdf"), "w") as f:
        f.write(URDF_MESH.format(name="rock", mesh="rock.obj", scale="1.5 1.0 0.8"))
    with open(os.path.join(folder, "ball.urdf"), "w") as f:
        f.write(URDF_SPHERE.format(r=0.4))
    return folder


def mesh_env_cfg(folder, num_assets=4):
    """dynamic_env with its objects drawn from `folder` (meshes and spheres only)"""
    from aerial_gym_simulator_b200.config import asset_config as AC
    from aerial_gym_simulator_b200.config.env_config import DynamicEnvironmentCfg

    params = type("mesh_asset_params", (AC.dynamic_object_asset_params,), dict(asset_folder=folder, num_assets=num_assets))

    class Cfg(DynamicEnvironmentCfg):
        class env_config(DynamicEnvironmentCfg.env_config):
            include_asset_type = {"objects": True}
            asset_type_to_dict_map = {"objects": params}
    return Cfg

