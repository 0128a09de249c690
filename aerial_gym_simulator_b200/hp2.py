"""Host side of HP2 (ray-cast sensors): device tensors + C-ABI calls, no hot-path arithmetic.

``RayScene``  replaces WarpEnv (env_manager/warp_env_manager.py): per-env triangle scene + BVH,
              rebuilt on reset from the asset root poses.
``RaySensor`` replaces WarpSensor/WarpCam/WarpLidar (sensors/warp/warp_sensor.py, warp_cam.py,
              warp_lidar.py): one camera or LiDAR type mounted on every robot.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Optional, Sequence

import numpy as np
import torch

from . import _lib
from ._lib import AgxHp2Scene, AgxHp2Sensor


def box_triangles(size: Sequence[float]) -> np.ndarray:
    """[12,9] object-frame triangles (v0,v1,v2) of a URDF <box size="x y z"/> centred at the origin:
    the mesh the reference obtains through urdfpy/trimesh for every shipped obstacle
    (assets/warp_asset.py:23-60; resources/models/environment_assets/{objects,panels,walls})."""
    hx, hy, hz = (float(s) / 2.0 for s in size)
    v = np.array([[-hx, -hy, -hz], [-hx, -hy, hz], [-hx, hy, -hz], [-hx, hy, hz],
                  [hx, -hy, -hz], [hx, -hy, hz], [hx, hy, -hz], [hx, hy, hz]], dtype=np.float32)
    f = np.array([[1, 3, 0], [4, 1, 0], [0, 3, 2], [2, 4, 0], [1, 7, 3], [5, 1, 4],
                  [5, 7, 1], [3, 7, 2], [6, 4, 2], [2, 7, 6], [6, 5, 4], [7, 5, 6]])
    return v[f].reshape(12, 9).astype(np.float32)


def box_obb(size: Sequence[float], R=None, p=None) -> np.ndarray:
    """[16] oriented-box record of a box template: centre, 3 axes (columns of R), half extents, kind.
    kind = 2: the template's triangles are box_triangles(size) in that order, transformed by (R, p) --
    the ray-caster may then test only the two triangles of the face a ray enters through; kind = 1: some
    other mesh with this bounding box (culling only); kind = 0: no box."""
    R = np.eye(3) if R is None else np.asarray(R, dtype=np.float64)
    p = np.zeros(3) if p is None else np.asarray(p, dtype=np.float64)
    return np.concatenate([p, R[:, 0], R[:, 1], R[:, 2], np.asarray(size, dtype=np.float64) / 2.0, [2.0]]).astype(np.float32)


def cylinder_triangles(radius: float, length: float, sections: int = 32) -> np.ndarray:
    """[4*sections,9] object-frame triangles of a URDF <cylinder radius length/> (axis = z, centred): a `sections`-gon prism with fan
    caps -- what the reference obtains through urdfpy -> trimesh.creation.cylinder (a revolved rectangle, 32 sections by default;
    assets/warp_asset.py:19-24).  trimesh is not installable here: vertex angles 2 pi k / sections are the published construction,
    parity against trimesh's own tessellation unpinned."""
    r, h = float(radius), float(length) / 2.0
    ang = 2.0 * np.pi * np.arange(sections) / sections
    ring = np.stack([r * np.cos(ang), r * np.sin(ang)], axis=1)
    tris = []
    for k in range(sections):
        a, b = ring[k], ring[(k + 1) % sections]
        lo_a, lo_b, hi_a, hi_b = (a[0], a[1], -h), (b[0], b[1], -h), (a[0], a[1], h), (b[0], b[1], h)
        tris.append(((0.0, 0.0, -h), lo_b, lo_a))   # bottom cap (outward normal -z)
        tris.append((lo_a, lo_b, hi_b))             # side
        tris.append((lo_a, hi_b, hi_a))
        tris.append(((0.0, 0.0, h), hi_a, hi_b))    # top cap (+z)
    return np.asarray(tris, dtype=np.float32).reshape(-1, 9)


def icosphere_triangles(radius: float, subdivisions: int = 3) -> np.ndarray:
    """[20*4^s,9] object-frame triangles of a URDF <sphere radius/>: what urdfpy obtains from trimesh.creation.icosphere (3
    subdivisions: 642 vertices, 1280 faces).  Restated from the published construction: the regular icosahedron, each face split
    into four at its edge midpoints (a, ab, ca | ab, b, bc | ca, bc, c | ab, bc, ca), shared midpoints merged, every vertex
    projected onto the sphere.  Parity against trimesh's own vertex order unpinned, as for cylinder_triangles."""
    t = (1.0 + math.sqrt(5.0)) / 2.0
    v = [[-1, t, 0], [1, t, 0], [-1, -t, 0], [1, -t, 0], [0, -1, t], [0, 1, t], [0, -1, -t], [0, 1, -t],
         [t, 0, -1], [t, 0, 1], [-t, 0, -1], [-t, 0, 1]]
    v = [np.asarray(x, np.float64) / np.linalg.norm(x) for x in v]
    f = [(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4), (11, 10, 2), (10, 7, 6), (7, 1, 8),
         (3, 9, 4), (3, 4, 2), (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11), (6, 2, 10), (8, 6, 7), (9, 8, 1)]
    for _ in range(subdivisions):
        mid = {}

        def m(i, j):
            key = (min(i, j), max(i, j))
            if key not in mid:
                c = v[i] + v[j]
                mid[key] = len(v)
                v.append(c / np.linalg.norm(c))
            return mid[key]

        nf = []
        for a, b, c in f:
            ab, bc, ca = m(a, b), m(b, c), m(c, a)
            nf += [(a, ab, ca), (ab, b, bc), (ca, bc, c), (ab, bc, ca)]
        f = nf
    return (np.asarray(v)[np.asarray(f)] * float(radius)).reshape(-1, 9).astype(np.float32)


BLAS_LEAF_TRIS = 4


def build_blas(tris) -> dict:
    """Bottom-level BVH of one mesh template, built once on the host, deterministic: breadth-first binary tree, every node
    splits its triangles at the median of their centroids along the longest axis of the centroid bounds (stable sort, so ties
    keep file order), leaves of <= BLAS_LEAF_TRIS triangles.  The median split bounds the depth by log2(n / BLAS_LEAF_TRIS) + 1.
    Returns order [n] (file index of each leaf-order triangle), topo [N,2] ((first child, 0) internal / (first triangle, count)
    leaf), levels [AGX_HP2_BLAS_MAX_DEPTH + 1] (nodes of depth d are levels[d]:levels[d+1])."""
    t = np.asarray(tris, np.float32).reshape(-1, 3, 3).astype(np.float64)
    n = len(t)
    if n < 1:
        raise ValueError("a mesh needs at least one triangle")
    cent = t.mean(axis=1)
    order = np.arange(n)
    nodes, topo, depth = [(0, n, 0)], [], []
    i = 0
    while i < len(nodes):
        a, b, d = nodes[i]
        depth.append(d)
        if b - a <= BLAS_LEAF_TRIS:
            topo.append((a, b - a))
        else:
            c = cent[order[a:b]]
            ax = int(np.argmax(c.max(axis=0) - c.min(axis=0)))
            order[a:b] = order[a:b][np.argsort(c[:, ax], kind="stable")]
            mid = a + (b - a) // 2
            topo.append((len(nodes), 0))
            nodes += [(a, mid, d + 1), (mid, b, d + 1)]
        i += 1
    D = _lib.BLAS_MAX_DEPTH
    if max(depth) >= D:
        raise ValueError(f"mesh of {n} triangles: BLAS deeper than {D} levels")
    levels = np.searchsorted(np.asarray(depth), np.arange(D + 1), side="left").astype(np.int32)
    return dict(order=order.astype(np.int32), topo=np.asarray(topo, np.int32).reshape(-1, 2), levels=levels)


def _next_pow2(v: int) -> int:
    p = 1
    while p < v:
        p <<= 1
    return p


class RayScene:
    """templates: list of [n_i,9] float32 triangle arrays (n_i <= tris_per_object; split bigger
    meshes into several templates sharing a pose).  obj_template / obj_seg_counter: int [E,K].
    obj_pose: float32 device tensor [E,K,>=7] (e.g. env_asset_state_tensor, a view is fine as long
    as the last dim is contiguous and rows are uniformly strided).
    mesh_templates: list of [n_m,9] triangle arrays of any size (URDF <mesh> / <sphere> visuals); template index
    len(templates) + m in obj_template.  Each such object is one mesh object with its own bottom-level BVH (build_blas);
    its face ids follow the array's order.  tmpl_seg_base / tmpl_seg_mask (and tmpl_obb, zero rows for meshes) cover
    templates + mesh_templates."""

    def __init__(self, templates, tmpl_seg_base, tmpl_seg_mask, obj_template, obj_seg_counter, obj_pose: torch.Tensor,
                 device="cuda:0", tris_per_object: Optional[int] = None, bounds_min=None, bounds_max=None, tmpl_obb=None,
                 mesh_templates=None):
        """tmpl_obb: optional [T,16] oriented-box records (box_obb) of the templates that ARE boxes (valid=1);
        purely a culling aid -- results are identical with or without it."""
        self.lib = _lib.load()
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise _lib.AgxError("RayScene needs a CUDA device: there is no CPU path")
        dev = self.device
        obj_template = np.asarray(obj_template, dtype=np.int32)
        E, K = obj_template.shape
        meshes = [np.asarray(t, np.float32).reshape(-1, 9) for t in (mesh_templates or [])]
        nT, M = len(templates), len(meshes)
        L = int(tris_per_object or max([len(t) for t in templates] or [1]))
        if any(len(t) > L for t in templates):
            raise ValueError("template larger than tris_per_object: split it on the host")
        if len(tmpl_seg_base) != nT + M or len(tmpl_seg_mask) != nT + M:
            raise ValueError("tmpl_seg_base / tmpl_seg_mask need one entry per template and mesh template")
        if obj_template.min() < 0 or obj_template.max() >= nT + M:
            raise ValueError("obj_template out of range")
        offs = np.zeros(nT + M + 1, dtype=np.int32)  # mesh templates have no cluster triangles
        offs[1:nT + 1] = np.cumsum([len(t) for t in templates])
        offs[nT + 1:] = offs[nT]
        pad = [] if offs[nT] else [np.zeros(1, np.int32)]  # a scene of mesh objects only: keep the cluster tables non-empty
        tris = np.concatenate([np.asarray(t, np.float32).reshape(-1, 9) for t in templates] + [np.zeros((len(pad), 9), np.float32)], axis=0)
        seg_base = np.concatenate([np.broadcast_to(np.asarray(b, np.int32), (len(t),)) for b, t in zip(tmpl_seg_base, templates)] + pad)
        seg_mask = np.concatenate([np.broadcast_to(np.asarray(m, np.int32), (len(t),)) for m, t in zip(tmpl_seg_mask, templates)] + pad)
        T = lambda a, dt: torch.tensor(np.ascontiguousarray(a), dtype=dt, device=dev)
        self.E, self.K, self.L, self.P = E, K, L, _next_pow2(K)
        self.tmpl_tri_offset = T(offs, torch.int32)
        self.tmpl_tris = T(tris, torch.float32)
        self.tmpl_seg_base = T(seg_base, torch.int32)
        self.tmpl_seg_mask = T(seg_mask, torch.int32)
        self.obj_template = T(obj_template, torch.int32)
        self.obj_seg_counter = T(np.asarray(obj_seg_counter, np.int32), torch.int32)
        self.obj_pose = obj_pose
        if obj_pose.device != dev or obj_pose.dtype != torch.float32 or obj_pose.shape[:2] != (E, K) or obj_pose.shape[2] < 7:
            raise ValueError("obj_pose must be float32 [E,K,>=7] on the scene's device")
        if obj_pose.stride(2) != 1 or obj_pose.stride(0) != K * obj_pose.stride(1):
            raise ValueError("obj_pose rows must be uniformly strided with a contiguous last dim")
        self.bounds_min, self.bounds_max = bounds_min, bounds_max
        nb = lambda which: int(self.lib.agx_hp2_scene_bytes(K, L, which))
        self.tris = torch.zeros(E * nb(0) // 4, dtype=torch.float32, device=dev)
        self.nodes = torch.zeros(E * nb(1) // 4, dtype=torch.float32, device=dev)
        self.leaf_object = torch.full((E * nb(2) // 4,), -1, dtype=torch.int32, device=dev)
        self.face_offset = torch.zeros(E * K, dtype=torch.int32, device=dev)
        self.tmpl_obb = self.obb = None
        if tmpl_obb is not None:
            tmpl_obb = np.asarray(tmpl_obb, dtype=np.float32).reshape(nT + M, 16)
            self.tmpl_obb = T(tmpl_obb, torch.float32)
            self.obb = torch.zeros(E * K * 16, dtype=torch.float32, device=dev)
        s = AgxHp2Scene()
        s.num_envs, s.num_objects, s.leaves_pow2, s.tris_per_object = E, K, self.P, L
        s.num_templates, s.obj_pose_stride = nT + M, obj_pose.stride(1)
        for name in ("tmpl_tri_offset", "tmpl_tris", "tmpl_seg_base", "tmpl_seg_mask", "obj_pose", "obj_template",
                     "obj_seg_counter", "tris", "nodes", "leaf_object", "face_offset"):
            setattr(s, name, getattr(self, name).data_ptr())
        s.tmpl_obb = self.tmpl_obb.data_ptr() if self.tmpl_obb is not None else None
        s.obb = self.obb.data_ptr() if self.obb is not None else None
        s.bounds_min = bounds_min.data_ptr() if bounds_min is not None else None
        s.bounds_max = bounds_max.data_ptr() if bounds_max is not None else None
        if M:
            self._set_meshes(s, meshes, tmpl_seg_base[nT:], tmpl_seg_mask[nT:], obj_template, nT)
        self.c = s

    def _set_meshes(self, s, meshes, seg_base, seg_mask, obj_template, T):
        """device tables of the mesh templates (one BLAS each) and the per-env mesh slabs"""
        dev, M, (E, K) = self.device, len(meshes), obj_template.shape
        T_ = lambda a, dt: torch.tensor(np.ascontiguousarray(a), dtype=dt, device=dev)
        blas = [build_blas(m) for m in meshes]
        n_tri = np.array([len(m) for m in meshes], np.int64)
        n_node = np.array([len(b["topo"]) for b in blas], np.int64)
        mesh_of = np.full(T + M, -1, np.int32)
        mesh_of[T:] = np.arange(M)
        om = mesh_of[obj_template]  # [E,K]
        is_mesh = om >= 0
        cnt_t = np.where(is_mesh, n_tri[np.maximum(om, 0)], 0)
        cnt_n = np.where(is_mesh, n_node[np.maximum(om, 0)], 0)
        slot = np.stack([np.cumsum(cnt_t, axis=1) - cnt_t, np.cumsum(cnt_n, axis=1) - cnt_n], axis=-1)
        slot[~is_mesh] = -1
        per_t, per_n = max(int(cnt_t.sum(axis=1).max()), 1), max(int(cnt_n.sum(axis=1).max()), 1)
        if per_t * E * 48 > 2 ** 40 or per_t >= 2 ** 31:
            raise ValueError("mesh storage too large")
        self.tmpl_mesh = T_(mesh_of, torch.int32)
        self.mesh_tri_offset = T_(np.concatenate([[0], np.cumsum(n_tri)]), torch.int32)
        self.mesh_tris = T_(np.concatenate([m[b["order"]] for m, b in zip(meshes, blas)]), torch.float32)
        self.mesh_tri_index = T_(np.concatenate([b["order"] for b in blas]), torch.int32)
        self.mesh_seg = T_(np.stack([np.asarray(seg_base, np.int32), np.asarray(seg_mask, np.int32)], axis=1), torch.int32)
        self.mesh_node_offset = T_(np.concatenate([[0], np.cumsum(n_node)]), torch.int32)
        self.mesh_topo = T_(np.concatenate([b["topo"] for b in blas]), torch.int32)
        self.mesh_levels = T_(np.stack([b["levels"] for b in blas]), torch.int32)
        self.obj_mesh_slot = T_(slot, torch.int32)
        self.mesh_world_tris = torch.zeros(E * per_t * 12, dtype=torch.float32, device=dev)
        self.mesh_world_nodes = torch.zeros(E * per_n * 8, dtype=torch.float32, device=dev)
        s.num_meshes, s.mesh_tris_per_env, s.mesh_nodes_per_env = M, per_t, per_n
        for name in ("tmpl_mesh", "mesh_tri_offset", "mesh_tris", "mesh_tri_index", "mesh_seg", "mesh_node_offset", "mesh_topo",
                     "mesh_levels", "obj_mesh_slot", "mesh_world_tris", "mesh_world_nodes"):
            setattr(s, name, getattr(self, name).data_ptr())

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def update(self, mask: Optional[torch.Tensor] = None):
        """Re-transform + rebuild the BVH of the masked envs (all when mask is None)."""
        if mask is not None and (mask.dtype != torch.bool or mask.shape != (self.E,)):
            raise ValueError("mask must be bool [E]")
        m = C.c_void_p(mask.data_ptr()) if mask is not None else None
        _lib.check(self.lib.agx_hp2_update_scene(C.byref(self.c), m, self._stream()), "agx_hp2_update_scene")


    def collide(self, robot_state: torch.Tensor, radius: float, crashes: torch.Tensor, min_dist: Optional[torch.Tensor] = None):
        """crashes (bool [E]) |= robot collision sphere overlaps the env mesh (row a14)."""
        if crashes.dtype != torch.bool or crashes.shape != (self.E,):
            raise ValueError("crashes must be bool [E]")
        if robot_state.shape[0] != self.E or robot_state.stride(1) != 1:
            raise ValueError("robot_state must be [E,>=3] with contiguous rows")
        md = C.c_void_p(min_dist.data_ptr()) if min_dist is not None else None
        _lib.check(self.lib.agx_hp2_collide(C.byref(self.c), C.c_void_p(robot_state.data_ptr()), robot_state.stride(0),
                                            C.c_float(radius), C.c_void_p(crashes.data_ptr()), md, self._stream()),
                   "agx_hp2_collide")

    def contact(self, robot_state: torch.Tensor, params: _lib.AgxContactParams, force: torch.Tensor, crashes: torch.Tensor,
                contact_obj: Optional[torch.Tensor] = None, motion: Optional["ContactMotion"] = None,
                mass: Optional["ObstacleMass"] = None):
        """One rigid-contact solve against this scene (and the ground plane if params.ground_plane): see contact()."""
        contact(self, robot_state, params, force, crashes, contact_obj, motion, mass)


class ContactMotion:
    """What the moving-obstacle contact solve (agx_hp2_contact_moving) reads of the obstacles.
    asset_state: float32 [E,A,>=13] device tensor (env_asset_state_tensor: x y z, q xyzw, world linear and angular velocity per
    asset), rows uniformly strided with a contiguous last dim; read at every solve, so it may change between solves.
    obj_asset: integer [E,K]: the asset each scene object belongs to, every value in [0, A).  Checked here once (one host read), so
    that the solves themselves never synchronise with the host; kept as a contiguous int32 device copy."""

    def __init__(self, asset_state: torch.Tensor, obj_asset: torch.Tensor):
        if not isinstance(asset_state, torch.Tensor) or asset_state.dtype != torch.float32 or asset_state.dim() != 3 \
                or asset_state.shape[2] < 13 or asset_state.shape[1] < 1:
            raise ValueError("asset_state must be a float32 [E,A>=1,>=13] tensor")
        if asset_state.stride(2) != 1 or asset_state.stride(0) != asset_state.shape[1] * asset_state.stride(1):
            raise ValueError("asset_state rows must be uniformly strided with a contiguous last dim")
        if not isinstance(obj_asset, torch.Tensor) or obj_asset.dtype not in (torch.int32, torch.int64) or obj_asset.dim() != 2 \
                or obj_asset.shape[0] != asset_state.shape[0] or obj_asset.device != asset_state.device:
            raise ValueError("obj_asset must be an integer [E,K] tensor on asset_state's device, E = asset_state.shape[0]")
        A = asset_state.shape[1]
        if obj_asset.numel() and (int(obj_asset.min()) < 0 or int(obj_asset.max()) >= A):
            raise ValueError(f"obj_asset values must be in [0, {A})")
        self.asset_state, self.obj_asset = asset_state, obj_asset.to(torch.int32).contiguous()
        self.E, self.K, self.device = obj_asset.shape[0], obj_asset.shape[1], asset_state.device
        self.c = _lib.AgxContactMotion(asset_state=asset_state.data_ptr(), asset_stride=asset_state.stride(1), num_assets=A,
                                       obj_asset=self.obj_asset.data_ptr())


class ObstacleMass:
    """The per-(env, asset) mass table of the dynamic-obstacle contact solve (agx_hp2_contact_dynamic), one AgxObstacleMass per row.
    table: float32 [E,A,13] contiguous device tensor: inverse mass, COM in the asset frame (3), inverse inertia about the COM in
    asset-frame axes (9, row-major).  Checked here once (one host read): finite values, inverse mass >= 0.  An all-zero row is a
    kinematic asset (infinite mass: the solve reads its twist and never writes its row)."""

    def __init__(self, table: torch.Tensor):
        if not isinstance(table, torch.Tensor) or table.dtype != torch.float32 or table.dim() != 3 or table.shape[2] != 13 \
                or table.shape[1] < 1:
            raise ValueError("the obstacle mass table must be a float32 [E,A>=1,13] tensor")
        if not table.is_contiguous():
            raise ValueError("the obstacle mass table must be contiguous")
        if not bool(torch.isfinite(table).all()):
            raise ValueError("the obstacle mass table must be finite")
        if bool((table[..., 0] < 0).any()):
            raise ValueError("obstacle inverse masses must be >= 0")
        self.table, self.E, self.A, self.device = table, table.shape[0], table.shape[1], table.device

    @staticmethod
    def row(mass: float, com, inertia) -> np.ndarray:
        """one float32 row from a mass, a COM (asset frame) and an inertia about the COM (asset-frame axes)"""
        return np.concatenate([[1.0 / mass], np.asarray(com, np.float64).reshape(3),
                               np.linalg.inv(np.asarray(inertia, np.float64).reshape(3, 3)).reshape(9)]).astype(np.float32)


class ObstacleHull:
    """The vertex table of the obstacle–ground contact (agx_obstacle_ground_contact), one AgxObstacleHull.
    vertices: float32 [V,3], the asset-frame vertices of every file, file after file; file_offset: integer [F+1], file f's vertices
    are vertices[file_offset[f]:file_offset[f+1]]; file_reach: float32 [F], each >= the largest distance of the file's vertices from
    the asset origin; asset_file: integer [E,A], the file of each (env, asset).  Checked here once (one host read): finite values,
    offsets from 0, non-decreasing and ending at V, every asset_file in [0, F).  Kept as contiguous copies on vertices' device
    (int32 indices)."""

    def __init__(self, vertices: torch.Tensor, file_offset: torch.Tensor, file_reach: torch.Tensor, asset_file: torch.Tensor):
        for name, x, fp in (("vertices", vertices, True), ("file_offset", file_offset, False), ("file_reach", file_reach, True),
                            ("asset_file", asset_file, False)):
            if not isinstance(x, torch.Tensor) or x.is_floating_point() != fp or x.dtype == torch.bool or x.is_complex():
                raise ValueError(f"{name} must be a{' floating-point' if fp else 'n integer'} tensor")
        dev = vertices.device
        v, off, reach, af = (x.to(device=dev, dtype=dt).contiguous() for x, dt in (
            (vertices, torch.float32), (file_offset, torch.int32), (file_reach, torch.float32), (asset_file, torch.int32)))
        if v.dim() != 2 or v.shape[1] != 3:
            raise ValueError("vertices must be [V,3]")
        if reach.dim() != 1 or reach.shape[0] < 1 or off.shape != (reach.shape[0] + 1,):
            raise ValueError("file_reach must be [F>=1] and file_offset [F+1]")
        if af.dim() != 2 or af.shape[1] < 1:
            raise ValueError("asset_file must be [E,A>=1]")
        F, V = reach.shape[0], v.shape[0]
        checks = torch.stack([torch.isfinite(v).all(), torch.isfinite(reach).all(), (reach >= 0).all(), off[0] == 0, off[-1] == V,
                              (off[1:] >= off[:-1]).all(), (af >= 0).all(), (af < F).all()]).cpu()
        msgs = ("vertices must be finite", "file_reach must be finite", "file_reach must be >= 0", "file_offset must start at 0",
                f"file_offset must end at V = {V}", "file_offset must be non-decreasing", f"asset_file values must be in [0, {F})",
                f"asset_file values must be in [0, {F})")
        for ok, msg in zip(checks.tolist(), msgs):
            if not ok:
                raise ValueError(msg)
        self.vertices, self.file_offset, self.file_reach, self.asset_file = v, off, reach, af
        self.E, self.A, self.F, self.device = af.shape[0], af.shape[1], F, v.device
        self.c = _lib.AgxObstacleHull(vertices=v.data_ptr(), file_offset=off.data_ptr(), file_reach=reach.data_ptr(),
                                      asset_file=af.data_ptr(), num_files=F)

    @classmethod
    def from_files(cls, file_vertices, asset_file, device):
        """from a list of per-file vertex arrays ([n,3], asset frame) and the [E,A] file index; each file's reach is the largest
        distance of its vertices from the origin, rounded up to the next float32"""
        vs = [np.asarray(x, np.float32).reshape(-1, 3) for x in file_vertices]
        reach = np.array([np.sqrt((x.astype(np.float64) ** 2).sum(1)).max() if len(x) else 0.0 for x in vs], np.float32)
        reach = np.nextafter(reach, np.float32(np.inf))
        off = np.concatenate([[0], np.cumsum([len(x) for x in vs])]).astype(np.int32)
        v = np.concatenate(vs) if vs else np.zeros((0, 3), np.float32)
        return cls(*(torch.from_numpy(np.ascontiguousarray(x)).to(device) for x in (v, off, reach, np.asarray(asset_file))))


class ObstacleBoxes:
    """The box table of the obstacle–obstacle contact (agx_obstacle_obstacle_contact), one AgxObstacleBoxes.
    boxes: float32 [F,15], each file's box in the asset frame: centre (3), the three unit axes (3 each; box_obb's layout), the half
    extents (3); asset_file: integer [E,A], the file of each (env, asset).  Checked here once (one host read): finite values, half
    extents >= 0, axes orthonormal to 1e-5, every asset_file in [0, F).  Kept as contiguous copies on boxes' device (int32 indices)."""

    def __init__(self, boxes: torch.Tensor, asset_file: torch.Tensor):
        for name, x, fp in (("boxes", boxes, True), ("asset_file", asset_file, False)):
            if not isinstance(x, torch.Tensor) or x.is_floating_point() != fp or x.dtype == torch.bool or x.is_complex():
                raise ValueError(f"{name} must be a{' floating-point' if fp else 'n integer'} tensor")
        dev = boxes.device
        b = boxes.to(device=dev, dtype=torch.float32).contiguous()
        af = asset_file.to(device=dev, dtype=torch.int32).contiguous()
        if b.dim() != 2 or b.shape[0] < 1 or b.shape[1] != 15:
            raise ValueError("boxes must be [F>=1,15]")
        if af.dim() != 2 or af.shape[1] < 1:
            raise ValueError("asset_file must be [E,A>=1]")
        F = b.shape[0]
        ax = b[:, 3:12].double().view(F, 3, 3)
        gram = ax @ ax.transpose(1, 2)
        checks = torch.stack([torch.isfinite(b).all(), (b[:, 12:15] >= 0).all(),
                              ((gram - torch.eye(3, dtype=gram.dtype, device=dev)).abs() <= 1e-5).all(),
                              (af >= 0).all(), (af < F).all()]).cpu()
        msgs = ("boxes must be finite", "box half extents must be >= 0", "box axes must be orthonormal",
                f"asset_file values must be in [0, {F})", f"asset_file values must be in [0, {F})")
        for ok, msg in zip(checks.tolist(), msgs):
            if not ok:
                raise ValueError(msg)
        self.boxes, self.asset_file = b, af
        self.E, self.A, self.F, self.device = af.shape[0], af.shape[1], F, dev
        self.c = _lib.AgxObstacleBoxes(boxes=b.data_ptr(), asset_file=af.data_ptr(), num_files=F)

    @staticmethod
    def row(obb) -> np.ndarray:
        """the [15] table row of a box from its box_obb record (centre, axes, half extents; the kind is dropped)"""
        return np.asarray(obb, np.float32)[0:15].copy()


def obstacle_obstacle_contact(params: _lib.AgxContactParams, motion: ContactMotion, mass: ObstacleMass, boxes: ObstacleBoxes):
    """agx_obstacle_obstacle_contact: the free obstacle assets of motion.asset_state [E,A,>=13] against each other, one oriented box
    each (boxes); the rows with a contact get their new twist and position correction in place.  A <= 64.  Of params only
    contact_offset, rest_offset, dt, friction, max_depenetration_velocity and iterations are read."""
    if not isinstance(params, _lib.AgxContactParams):
        raise ValueError("params must be an AgxContactParams")
    if not isinstance(motion, ContactMotion):
        raise ValueError("motion must be a ContactMotion")
    if not isinstance(mass, ObstacleMass):
        raise ValueError("mass must be an ObstacleMass")
    if not isinstance(boxes, ObstacleBoxes):
        raise ValueError("boxes must be an ObstacleBoxes")
    st = motion.asset_state
    dev = st.device
    E, A = st.shape[0], st.shape[1]
    if (mass.E, mass.A) != (E, A) or mass.device != dev:
        raise ValueError("mass must have one row per motion asset [E,A], on the asset rows' device")
    if (boxes.E, boxes.A) != (E, A) or boxes.device != dev:
        raise ValueError("boxes must have one file index per motion asset [E,A], on the asset rows' device")
    if A > _lib.OBSTACLE_MAX_ASSETS:
        raise ValueError(f"obstacle_obstacle_contact takes at most {_lib.OBSTACLE_MAX_ASSETS} assets per env, not {A}")
    if dev.type != "cuda":
        raise _lib.AgxError("obstacle_obstacle_contact needs a CUDA device: there is no CPU path")
    _lib.check(_lib.load().agx_obstacle_obstacle_contact(E, A, C.byref(params), C.c_void_p(st.data_ptr()), st.stride(1),
                                                         C.c_void_p(mass.table.data_ptr()), C.byref(boxes.c),
                                                         C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
               "agx_obstacle_obstacle_contact")


def obstacle_ground_contact(params: _lib.AgxContactParams, motion: ContactMotion, mass: ObstacleMass, hull: ObstacleHull):
    """agx_obstacle_ground_contact: every free obstacle asset of motion.asset_state [E,A,>=13] against the ground plane z = 0 through
    the vertices of its file in hull; the rows with a kept contact get their new twist and position correction in place.  Of params
    only contact_offset, rest_offset, dt, friction, max_depenetration_velocity and iterations are read."""
    if not isinstance(params, _lib.AgxContactParams):
        raise ValueError("params must be an AgxContactParams")
    if not isinstance(motion, ContactMotion):
        raise ValueError("motion must be a ContactMotion")
    if not isinstance(mass, ObstacleMass):
        raise ValueError("mass must be an ObstacleMass")
    if not isinstance(hull, ObstacleHull):
        raise ValueError("hull must be an ObstacleHull")
    st = motion.asset_state
    dev = st.device
    E, A = st.shape[0], st.shape[1]
    if (mass.E, mass.A) != (E, A) or mass.device != dev:
        raise ValueError("mass must have one row per motion asset [E,A], on the asset rows' device")
    if (hull.E, hull.A) != (E, A) or hull.device != dev:
        raise ValueError("hull must have one file index per motion asset [E,A], on the asset rows' device")
    if dev.type != "cuda":
        raise _lib.AgxError("obstacle_ground_contact needs a CUDA device: there is no CPU path")
    _lib.check(_lib.load().agx_obstacle_ground_contact(E, A, C.byref(params), C.c_void_p(st.data_ptr()), st.stride(1),
                                                       C.c_void_p(mass.table.data_ptr()), C.byref(hull.c),
                                                       C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
               "agx_obstacle_ground_contact")


def contact(scene: Optional[RayScene], robot_state: torch.Tensor, params: _lib.AgxContactParams, force: torch.Tensor,
            crashes: torch.Tensor, contact_obj: Optional[torch.Tensor] = None, motion: Optional[ContactMotion] = None,
            mass: Optional[ObstacleMass] = None):
    """agx_hp2_contact: the robot's collision sphere against the scene's objects (scene None: none) and the ground plane.
    robot_state [E,>=13] float32: linear and world angular velocity updated in place; force [E,3] float32 = contact impulse / dt;
    crashes (bool [E]) |= |force| > params.force_threshold; contact_obj (int32 [E,CONTACT_MAX], optional) = contacts used.
    motion (ContactMotion of this scene's objects, optional): the obstacles move; the solve works on the robot's velocity relative to
    each obstacle's velocity at the contact point (agx_hp2_contact_moving).  None: every obstacle is at rest (agx_hp2_contact).
    mass (ObstacleMass of motion's assets, optional, needs motion): the obstacles are free bodies of that mass; every impulse also
    acts on the obstacle, and the touched free assets' rows of motion.asset_state are written back (agx_hp2_contact_dynamic)."""
    E = robot_state.shape[0]
    dev = robot_state.device
    if dev.type != "cuda":
        raise _lib.AgxError("contact needs a CUDA device: there is no CPU path")
    if scene is not None and (scene.E != E or scene.device != dev):
        raise ValueError("robot_state must have one row per scene env, on the scene's device")
    if robot_state.dtype != torch.float32 or robot_state.dim() != 2 or robot_state.shape[1] < 13 or robot_state.stride(1) != 1:
        raise ValueError("robot_state must be float32 [E,>=13] with contiguous rows")
    if crashes.dtype != torch.bool or crashes.shape != (E,) or crashes.device != dev:
        raise ValueError("crashes must be bool [E]")
    if force.dtype != torch.float32 or force.shape != (E, 3) or not force.is_contiguous() or force.device != dev:
        raise ValueError("force must be contiguous float32 [E,3]")
    if contact_obj is not None and (contact_obj.dtype != torch.int32 or contact_obj.shape != (E, _lib.CONTACT_MAX)
                                    or not contact_obj.is_contiguous() or contact_obj.device != dev):
        raise ValueError(f"contact_obj must be contiguous int32 [E,{_lib.CONTACT_MAX}]")
    if motion is not None:
        if not isinstance(motion, ContactMotion):
            raise ValueError("motion must be a ContactMotion")
        if scene is None:
            raise ValueError("moving obstacles need a scene")
        if (motion.E, motion.K) != (scene.E, scene.K) or motion.device != dev:
            raise ValueError("motion must map this scene's [E,K] objects, on the scene's device")
    if mass is not None:
        if not isinstance(mass, ObstacleMass):
            raise ValueError("mass must be an ObstacleMass")
        if motion is None:
            raise ValueError("dynamic obstacles need motion (their asset rows)")
        if (mass.E, mass.A) != tuple(motion.asset_state.shape[:2]) or mass.device != dev:
            raise ValueError("mass must have one row per motion asset [E,A], on the scene's device")
    lib = _lib.load()
    co = C.c_void_p(contact_obj.data_ptr()) if contact_obj is not None else None
    stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    if mass is not None:
        _lib.check(lib.agx_hp2_contact_dynamic(C.byref(scene.c), E, C.byref(params), C.byref(motion.c), C.c_void_p(mass.table.data_ptr()),
                                               C.c_void_p(robot_state.data_ptr()), robot_state.stride(0), C.c_void_p(force.data_ptr()),
                                               C.c_void_p(crashes.data_ptr()), co, stream), "agx_hp2_contact_dynamic")
        return
    if motion is not None:
        _lib.check(lib.agx_hp2_contact_moving(C.byref(scene.c), E, C.byref(params), C.byref(motion.c), C.c_void_p(robot_state.data_ptr()),
                                              robot_state.stride(0), C.c_void_p(force.data_ptr()), C.c_void_p(crashes.data_ptr()), co,
                                              stream), "agx_hp2_contact_moving")
        return
    _lib.check(lib.agx_hp2_contact(C.byref(scene.c) if scene is not None else None, E, C.byref(params),
                                   C.c_void_p(robot_state.data_ptr()), robot_state.stride(0), C.c_void_p(force.data_ptr()),
                                   C.c_void_p(crashes.data_ptr()), co, C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
               "agx_hp2_contact")


def camera_intrinsics(width, height, horizontal_fov_deg):
    """WarpCam.initialize_camera_matrices (sensors/warp/warp_cam.py:31-64): fp32 K, its inverse."""
    hf = math.radians(horizontal_fov_deg)
    u0, v0 = width / 2, height / 2
    f = width / 2 * 1 / math.tan(hf / 2)
    vfov = 2 * math.atan(height / (2 * f))
    au, av = u0 / math.tan(hf / 2), v0 / math.tan(vfov / 2)
    K = np.array([[au, 0, u0, 0], [0, av, v0, 0], [0, 0, 1, 0], [0, 0, 0, 1]], dtype=np.float32)
    Kinv = np.linalg.inv(K.astype(np.float64)).astype(np.float32)
    return Kinv[:3, :3].copy(), int(u0), int(v0)


def lidar_ray_table(height, width, hmin_deg, hmax_deg, vmin_deg, vmax_deg):
    """WarpLidar.initialize_ray_vectors (sensors/warp/warp_lidar.py:40-64)."""
    hmin, hmax = math.radians(hmin_deg), math.radians(hmax_deg)
    vmin, vmax = math.radians(vmin_deg), math.radians(vmax_deg)
    i = np.arange(height, dtype=np.float64)[:, None]
    j = np.arange(width, dtype=np.float64)[None, :]
    az = hmax - (hmax - hmin) * (j / (width - 1))
    el = vmax - (vmax - vmin) * (i / (height - 1))
    t = np.stack([np.cos(az) * np.cos(el), np.sin(az) * np.cos(el), np.sin(el) * np.ones_like(az)], axis=-1).astype(np.float32)
    n = np.sqrt((t ** 2).sum(-1, keepdims=True, dtype=np.float32))
    return (t / n).astype(np.float32)


def _quat_from_euler_deg(e):
    r, p, y = (math.radians(float(x)) for x in e)
    cy, sy, cr, sr, cp, sp = math.cos(y / 2), math.sin(y / 2), math.cos(r / 2), math.sin(r / 2), math.cos(p / 2), math.sin(p / 2)
    return [cy * sr * cp - sy * cr * sp, cy * cr * sp + sy * sr * cp, sy * cr * cp - cy * sr * sp, cy * cr * cp + sy * sr * sp]


class RaySensor:
    """cfg: a reference-style sensor config class (config/sensor_config/**): reads sensor_type,
    width, height, num_sensors, horizontal_fov_deg | *_fov_deg_min/max, max_range, min_range,
    calculate_depth, return_pointcloud, pointcloud_in_world_frame, segmentation_camera,
    normalize_range, far/near_out_of_range_value, euler_frame_rot_deg, sensor_noise."""

    def __init__(self, cfg, scene: RayScene, robot_state: torch.Tensor, pixels: torch.Tensor,
                 seg_pixels: Optional[torch.Tensor] = None, mount: Optional[torch.Tensor] = None):
        self.lib = _lib.load()
        self.cfg, self.scene = cfg, scene
        dev = scene.device
        E, S, H, W = scene.E, cfg.num_sensors, cfg.height, cfg.width
        st = cfg.sensor_type
        kinds = {"camera": _lib.SENSOR_CAMERA, "lidar": _lib.SENSOR_LIDAR, "stereo_camera": _lib.SENSOR_STEREO_CAMERA,
                 "normal_faceID_camera": _lib.SENSOR_NORMAL_FACEID_CAMERA, "normal_faceID_lidar": _lib.SENSOR_NORMAL_FACEID_LIDAR}
        if st not in kinds:
            raise NotImplementedError(f"sensor_type {st}")
        is_normal = st.startswith("normal_faceID")
        pc = bool(getattr(cfg, "return_pointcloud", False)) or is_normal
        want = (E, S, H, W, 3) if pc else (E, S, H, W)
        if tuple(pixels.shape) != want or pixels.dtype != torch.float32 or not pixels.is_contiguous():
            raise ValueError(f"pixels must be contiguous float32 {want}")
        if seg_pixels is not None and (tuple(seg_pixels.shape) != (E, S, H, W) or seg_pixels.dtype != torch.int32):
            raise ValueError("seg_pixels must be int32 [E,S,H,W]")
        if robot_state.shape[0] != E or robot_state.stride(1) != 1 or robot_state.shape[1] < 7:
            raise ValueError("robot_state must be [E,>=7] with contiguous rows")
        self.robot_state, self.pixels, self.seg_pixels = robot_state, pixels, seg_pixels
        if mount is None:  # identity mount
            mount = torch.zeros(E, S, 7, device=dev)
            mount[..., 6] = 1.0
        self.mount = mount.contiguous()
        noise = getattr(cfg, "sensor_noise", None)
        self.noise_enabled = bool(noise is not None and getattr(noise, "enable_sensor_noise", False))
        s = AgxHp2Sensor()
        s.kind = kinds[st]
        s.baseline = float(getattr(cfg, "baseline", 0.0))
        s.normal_in_world_frame = int(bool(getattr(cfg, "normal_in_world_frame", getattr(cfg, "pointcloud_in_world_frame", True))))
        s.width, s.height, s.num_sensors = W, H, S
        s.calculate_depth = int(bool(getattr(cfg, "calculate_depth", False)))
        s.return_pointcloud = int(pc and not is_normal)
        s.pointcloud_in_world_frame = int(bool(getattr(cfg, "pointcloud_in_world_frame", False)))
        s.segmentation = int(seg_pixels is not None)
        s.fuse_epilogue = int(not self.noise_enabled and not is_normal)  # limits only for camera/lidar/stereo (warp_sensor.py:198-200)
        s.normalize_range = int(bool(cfg.normalize_range))
        self.ray_table = None
        if "camera" in st:
            kinv, cx, cy = camera_intrinsics(W, H, cfg.horizontal_fov_deg)
            for i, v in enumerate(kinv.reshape(-1)):
                s.kinv[i] = float(v)
            s.c_x, s.c_y = cx, cy
        else:
            self.ray_table = torch.tensor(lidar_ray_table(H, W, cfg.horizontal_fov_deg_min, cfg.horizontal_fov_deg_max,
                                                          cfg.vertical_fov_deg_min, cfg.vertical_fov_deg_max), device=dev)
            s.ray_table = self.ray_table.data_ptr()
        s.far_plane = s.max_range = float(cfg.max_range)
        s.min_range = float(cfg.min_range)
        s.far_out_of_range_value = float(cfg.far_out_of_range_value)
        s.near_out_of_range_value = float(cfg.near_out_of_range_value)
        fq = torch.tensor(_quat_from_euler_deg(cfg.euler_frame_rot_deg), dtype=torch.float64).float()
        for i in range(4):
            s.frame_quat[i] = float(fq[i])
        s.robot_pose_stride = robot_state.stride(0)
        s.robot_pose, s.mount = robot_state.data_ptr(), self.mount.data_ptr()
        s.pixels = pixels.data_ptr()
        s.seg_pixels = seg_pixels.data_ptr() if seg_pixels is not None else None
        self.c = s

    def capture(self):
        """One launch: pose compose + ray gen + traversal + (range limits, normalise)."""
        _lib.check(self.lib.agx_hp2_cast(C.byref(self.scene.c), C.byref(self.c), self.scene._stream()), "agx_hp2_cast")
        return self.pixels

    def rays_per_frame(self):
        return self.scene.E * self.cfg.num_sensors * self.cfg.height * self.cfg.width
