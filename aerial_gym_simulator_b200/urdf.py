"""Minimal URDF reader: inertials, fixed-joint tree, box / cylinder / sphere / mesh visuals.

Replaces what the reference obtains from Isaac Gym asset properties
(robots/robot_manager.py:295-435: per-body mass / COM / inertia, body poses) and from
urdfpy + trimesh (assets/warp_asset.py:19-60: visual meshes with link transforms).
Only what the hot paths consume is parsed; there is no physics here."""
from __future__ import annotations

import math
import os
import xml.etree.ElementTree as ET
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import numpy as np


def rpy_to_matrix(rpy) -> np.ndarray:
    """URDF fixed-axis roll-pitch-yaw: R = Rz(yaw) Ry(pitch) Rx(roll)."""
    r, p, y = (float(v) for v in rpy)
    cr, sr, cp, sp, cy, sy = math.cos(r), math.sin(r), math.cos(p), math.sin(p), math.cos(y), math.sin(y)
    return np.array([
        [cy * cp, cy * sp * sr - sy * cr, cy * sp * cr + sy * sr],
        [sy * cp, sy * sp * sr + cy * cr, sy * sp * cr - cy * sr],
        [-sp, cp * sr, cp * cr],
    ])


def _vec(s: Optional[str], n=3, default=0.0):
    if s is None:
        return np.full(n, default)
    return np.array([float(x) for x in s.split()], dtype=np.float64)


@dataclass
class Visual:
    kind: str  # "box" | "sphere" | "cylinder" | "mesh"
    size: np.ndarray
    R: np.ndarray
    p: np.ndarray
    filename: Optional[str] = None


@dataclass
class Link:
    name: str
    mass: float = 0.0
    com: np.ndarray = field(default_factory=lambda: np.zeros(3))
    com_R: np.ndarray = field(default_factory=lambda: np.eye(3))
    inertia: np.ndarray = field(default_factory=lambda: np.zeros((3, 3)))
    visuals: List[Visual] = field(default_factory=list)
    collisions: List[Visual] = field(default_factory=list)


@dataclass
class Joint:
    name: str
    parent: str
    child: str
    R: np.ndarray
    p: np.ndarray
    kind: str = "fixed"
    axis: np.ndarray = field(default_factory=lambda: np.array([1.0, 0.0, 0.0]))  # <axis xyz>, joint frame, as written
    lower: float = 0.0  # <limit lower upper>: rad, m for a prismatic joint
    upper: float = 0.0
    damping: float = 0.0  # <dynamics damping>: N m s / rad, N s / m for a prismatic joint
    effort: float = 0.0  # <limit effort>: N m, N for a prismatic joint (0: none given)


MOVABLE_JOINTS = ("revolute", "continuous", "prismatic")


@dataclass
class ArticulatedBodies:
    """The links of a URDF merged across its fixed joints into rigid bodies (UrdfModel.articulation).  Body 0 is the root link's; body
    i >= 1 hangs on one movable joint (DOF i - 1) -- revolute, continuous or prismatic (joint_kinds) -- and its frame is the frame of
    that joint's child link.  Bodies are numbered in body_order()'s depth-first order, so every parent precedes its children."""
    links: List[str]             # the link each body's frame is, [B]
    parent: np.ndarray           # [B] int, parent body (-1 for body 0)
    joint_names: List[str]       # [B] ("" for body 0)
    joint_kinds: List[str]
    joint_R: np.ndarray          # [B,3,3] parent body frame -> body frame at q = 0
    joint_p: np.ndarray          # [B,3]
    axis: np.ndarray             # [B,3] unit, body frame
    lower: np.ndarray            # [B]
    upper: np.ndarray
    limited: np.ndarray          # [B] bool: revolute or prismatic with lower < upper (always, for prismatic)
    urdf_damping: np.ndarray     # [B] <dynamics damping>
    mass: np.ndarray             # [B]
    com: np.ndarray              # [B,3] body frame
    inertia: np.ndarray          # [B,3,3] about the COM, body axes
    link_body: Dict[str, int]    # body each link was merged into
    link_in_body: Dict[str, Tuple[np.ndarray, np.ndarray]]  # (R, p) of each link in its body's frame
    effort_limit: Optional[np.ndarray] = None  # [B] <limit effort>, N m or N (0: none; body 0: 0); None = zeros

    def __post_init__(self):
        if self.effort_limit is None:
            self.effort_limit = np.zeros(len(self.links))

    @property
    def num_bodies(self) -> int:
        return len(self.links)

    @property
    def num_dofs(self) -> int:
        return len(self.links) - 1


@dataclass
class UrdfModel:
    name: str
    links: Dict[str, Link]
    joints: List[Joint]
    root: str

    def body_order(self) -> List[str]:
        """Rigid-body index order used by the reference configs' application_mask
        (e.g. base_quad_config.py:163: bodies 1-4 arms, 5-8 motors): root first, then the
        children of each link in name order, depth first."""
        children: Dict[str, List[str]] = {}
        for j in self.joints:
            children.setdefault(j.parent, []).append(j.child)
        out: List[str] = []

        def visit(n):
            out.append(n)
            for c in sorted(children.get(n, [])):
                visit(c)

        visit(self.root)
        return out

    def link_transforms(self) -> Dict[str, Tuple[np.ndarray, np.ndarray]]:
        """(R, p) of every link frame in the root frame, joints at their zero position."""
        tf = {self.root: (np.eye(3), np.zeros(3))}
        pending = list(self.joints)
        while pending:
            progressed = False
            for j in list(pending):
                if j.parent in tf:
                    Rp, pp = tf[j.parent]
                    tf[j.child] = (Rp @ j.R, pp + Rp @ j.p)
                    pending.remove(j)
                    progressed = True
            if not progressed:
                raise ValueError("URDF joint graph is not a tree rooted at " + self.root)
        return tf

    def composite_inertia(self) -> Tuple[float, np.ndarray, np.ndarray]:
        """Total mass, COM (root frame) and inertia about the COM in root-frame axes: the
        parallel-axis accumulation of robots/robot_manager.py:313-426."""
        tf = self.link_transforms()
        m_tot, c_sum = 0.0, np.zeros(3)
        for l in self.links.values():
            R, p = tf[l.name]
            c_sum += l.mass * (p + R @ l.com)
            m_tot += l.mass
        com = c_sum / m_tot if m_tot > 0 else np.zeros(3)
        J = np.zeros((3, 3))
        for l in self.links.values():
            R, p = tf[l.name]
            Rl = R @ l.com_R
            d = (p + R @ l.com) - com
            J += Rl @ l.inertia @ Rl.T + l.mass * (float(d @ d) * np.eye(3) - np.outer(d, d))
        return m_tot, com, J

    def articulation(self, max_bodies: int = 16) -> ArticulatedBodies:
        """The merged body table of an articulated robot.  Each body's mass, COM and inertia are the parallel-axis accumulation of
        composite_inertia() over the links merged into it.  Joints other than fixed / revolute / continuous / prismatic, a prismatic
        joint without a <limit> with lower < upper, a zero <axis> and more than `max_bodies` bodies raise ValueError."""
        by_child = {j.child: j for j in self.joints}
        names, parent, jn, jk, jR, jp, ax, lo, hi, lim, dmp, eff = [], [], [], [], [], [], [], [], [], [], [], []
        link_body, link_in_body = {}, {}
        for name in self.body_order():
            j = by_child.get(name)
            if j is None or j.kind == "fixed":
                if j is None:
                    b, T = 0, (np.eye(3), np.zeros(3))
                    names.append(name); parent.append(-1); jn.append(""); jk.append("")
                    jR.append(np.eye(3)); jp.append(np.zeros(3)); ax.append(np.zeros(3))
                    lo.append(0.0); hi.append(0.0); lim.append(False); dmp.append(0.0); eff.append(0.0)
                else:
                    b = link_body[j.parent]
                    Rp, pp = link_in_body[j.parent]
                    T = (Rp @ j.R, pp + Rp @ j.p)
                link_body[name], link_in_body[name] = b, T
                continue
            if j.kind not in MOVABLE_JOINTS:
                raise ValueError(f"joint '{j.name}' is {j.kind}: articulated robots support revolute, continuous and prismatic joints only")
            if j.kind == "prismatic" and not j.lower < j.upper:
                raise ValueError(f"joint '{j.name}' is prismatic without a <limit> with lower < upper ({j.lower}, {j.upper}): a slide "
                                 "must be bounded")
            a = np.asarray(j.axis, dtype=np.float64)
            n = float(np.linalg.norm(a))
            if not n > 0:
                raise ValueError(f"joint '{j.name}' has a zero <axis>")
            Rp, pp = link_in_body[j.parent]
            link_body[name], link_in_body[name] = len(names), (np.eye(3), np.zeros(3))
            names.append(name); parent.append(link_body[j.parent]); jn.append(j.name); jk.append(j.kind)
            jR.append(Rp @ j.R); jp.append(pp + Rp @ j.p); ax.append(a / n)
            limited = j.kind in ("revolute", "prismatic") and j.lower < j.upper
            lo.append(float(j.lower)); hi.append(float(j.upper)); lim.append(limited); dmp.append(float(j.damping))
            if not j.effort >= 0:
                raise ValueError(f"joint '{j.name}' has a negative <limit effort> ({j.effort})")
            eff.append(float(j.effort))
        B = len(names)
        if B > max_bodies:
            raise ValueError(f"{B} bodies after merging the fixed joints: at most {max_bodies} are supported ({max_bodies - 1} DOFs)")
        mass, com, inertia = np.zeros(B), np.zeros((B, 3)), np.zeros((B, 3, 3))
        csum = np.zeros((B, 3))
        for name, b in link_body.items():
            l = self.links[name]
            R, p = link_in_body[name]
            mass[b] += l.mass
            csum[b] += l.mass * (p + R @ l.com)
        for b in range(B):
            com[b] = csum[b] / mass[b] if mass[b] > 0 else np.zeros(3)
        for name, b in link_body.items():
            l = self.links[name]
            R, p = link_in_body[name]
            Rl = R @ l.com_R
            d = (p + R @ l.com) - com[b]
            inertia[b] += Rl @ l.inertia @ Rl.T + l.mass * (float(d @ d) * np.eye(3) - np.outer(d, d))
        return ArticulatedBodies(names, np.asarray(parent, np.int64), jn, jk, np.asarray(jR), np.asarray(jp), np.asarray(ax),
                                 np.asarray(lo), np.asarray(hi), np.asarray(lim, bool), np.asarray(dmp), mass, com, inertia,
                                 link_body, link_in_body, np.asarray(eff, np.float64))


def _parse_geometry(el, base_dir) -> Optional[Visual]:
    geom = el.find("geometry")
    if geom is None:
        return None
    org = el.find("origin")
    R = rpy_to_matrix(_vec(org.get("rpy") if org is not None else None))
    p = _vec(org.get("xyz") if org is not None else None)
    b = geom.find("box")
    if b is not None:
        return Visual("box", _vec(b.get("size")), R, p)
    s = geom.find("sphere")
    if s is not None:
        return Visual("sphere", np.array([float(s.get("radius"))]), R, p)
    c = geom.find("cylinder")
    if c is not None:
        return Visual("cylinder", np.array([float(c.get("radius")), float(c.get("length"))]), R, p)
    m = geom.find("mesh")
    if m is not None:
        fn = m.get("filename", "")
        return Visual("mesh", _vec(m.get("scale"), default=1.0), R, p, fn if "://" in fn else os.path.join(base_dir, fn))
    return None


def parse_urdf(path: str) -> UrdfModel:
    root_el = ET.parse(path).getroot()
    base_dir = os.path.dirname(os.path.abspath(path))
    links: Dict[str, Link] = {}
    for le in root_el.findall("link"):
        l = Link(le.get("name"))
        ine = le.find("inertial")
        if ine is not None:
            m = ine.find("mass")
            l.mass = float(m.get("value")) if m is not None else 0.0
            org = ine.find("origin")
            if org is not None:
                l.com = _vec(org.get("xyz"))
                l.com_R = rpy_to_matrix(_vec(org.get("rpy")))
            ie = ine.find("inertia")
            if ie is not None:
                g = lambda k: float(ie.get(k, 0.0))
                l.inertia = np.array([[g("ixx"), g("ixy"), g("ixz")], [g("ixy"), g("iyy"), g("iyz")], [g("ixz"), g("iyz"), g("izz")]])
        for ve in le.findall("visual"):
            v = _parse_geometry(ve, base_dir)
            if v is not None:
                l.visuals.append(v)
        for ce in le.findall("collision"):
            v = _parse_geometry(ce, base_dir)
            if v is not None:
                l.collisions.append(v)
        links[l.name] = l
    joints: List[Joint] = []
    children = set()
    for je in root_el.findall("joint"):
        org = je.find("origin")
        R = rpy_to_matrix(_vec(org.get("rpy") if org is not None else None))
        p = _vec(org.get("xyz") if org is not None else None)
        j = Joint(je.get("name"), je.find("parent").get("link"), je.find("child").get("link"), R, p, je.get("type", "fixed"))
        ae, le, de = je.find("axis"), je.find("limit"), je.find("dynamics")
        if ae is not None and ae.get("xyz") is not None:
            j.axis = _vec(ae.get("xyz"))
        if le is not None:
            j.lower, j.upper = float(le.get("lower", 0.0)), float(le.get("upper", 0.0))
            j.effort = float(le.get("effort", 0.0))
        if de is not None:
            j.damping = float(de.get("damping", 0.0))
        joints.append(j)
        children.add(j.child)
    roots = [n for n in links if n not in children]
    if len(roots) != 1:
        raise ValueError(f"{path}: expected exactly one root link, found {roots}")
    return UrdfModel(root_el.get("name", ""), links, joints, roots[0])


def box_visual_triangles(model: UrdfModel, use_collision=False):
    """Per-link list of [12,9] root-frame triangle arrays for every <box> visual (the obstacle
    assets the reference ships are all boxes).  Returns [(link_name, triangles, obb16)]."""
    from .hp2 import box_obb, box_triangles

    tf = model.link_transforms()
    out = []
    for name in model.body_order():
        l = model.links[name]
        R, p = tf[name]
        for v in (l.collisions if use_collision else l.visuals):
            if v.kind != "box":
                continue
            t = box_triangles(v.size).reshape(-1, 3).astype(np.float64)
            t = (R @ (v.R @ t.T + v.p[:, None]) + p[:, None]).T
            out.append((name, t.reshape(-1, 9).astype(np.float32), box_obb(v.size, R @ v.R, R @ v.p + p)))
    return out


def _obj_triangles(path) -> np.ndarray:
    verts, tris = [], []
    with open(path, "r", errors="replace") as f:
        for line in f:
            tok = line.split()
            if not tok:
                continue
            if tok[0] == "v":
                verts.append([float(x) for x in tok[1:4]])
            elif tok[0] == "f":
                # "i", "i/t", "i//n", "i/t/n"; negative indices count back from the last vertex read so far
                idx = [int(t.split("/")[0]) for t in tok[1:]]
                idx = [i - 1 if i > 0 else len(verts) + i for i in idx]
                for j in range(1, len(idx) - 1):  # fan triangulation of a polygon
                    tris.append((idx[0], idx[j], idx[j + 1]))
    if not tris:
        raise ValueError(f"{path}: no faces")
    v = np.asarray(verts, dtype=np.float64)
    return v[np.asarray(tris)].reshape(-1, 9)


def _stl_triangles(path) -> np.ndarray:
    with open(path, "rb") as f:
        data = f.read()
    if len(data) >= 84:
        n = int(np.frombuffer(data, "<u4", 1, 80)[0])
        if len(data) == 84 + 50 * n:  # binary: header, count, n x (normal, 3 vertices, attribute)
            rec = np.frombuffer(data, np.dtype([("n", "<f4", 3), ("v", "<f4", 9), ("a", "<u2")]), n, 84)
            return rec["v"].astype(np.float64)
    if not data.lstrip().startswith(b"solid"):
        raise ValueError(f"{path}: neither binary nor ASCII STL")
    v = [[float(x) for x in line.split()[1:4]] for line in data.decode("ascii", "replace").splitlines() if line.split()[:1] == ["vertex"]]
    if not v or len(v) % 3:
        raise ValueError(f"{path}: malformed ASCII STL")
    return np.asarray(v, dtype=np.float64).reshape(-1, 9)


def load_mesh(path, scale=(1.0, 1.0, 1.0)) -> np.ndarray:
    """[n,9] float64 triangles (v0,v1,v2) of a Wavefront OBJ or STL (ASCII or binary) file, in the file's face order, vertices
    multiplied by `scale`.  Polygons are fan-triangulated.  trimesh's load-time processing (vertex merge, removal of degenerate
    faces) is not applied, so face i here is the file's face i.  Any other format, or a URI (package://...), raises ValueError."""
    if "://" in path:
        raise ValueError(f"mesh {path}: URIs are not resolved; give a path relative to the URDF or an absolute one")
    ext = os.path.splitext(path)[1].lower()
    if ext == ".obj":
        t = _obj_triangles(path)
    elif ext == ".stl":
        t = _stl_triangles(path)
    else:
        raise ValueError(f"mesh {path}: unsupported format (OBJ and STL are read)")
    return (t.reshape(-1, 3) * np.broadcast_to(np.asarray(scale, np.float64), (3,))).reshape(-1, 9)


def visual_parts(model: UrdfModel, use_collision=False, max_tris=12):
    """Every visual of the model as ray-cast scene parts: [(link_name, link_index, triangles [n,9] in the root frame, obb16 or None)].
    A box is one part (its 12 triangles + the oriented box the ray-caster uses for the entry-face shortcut, kind 2); a cylinder is
    tessellated (hp2.cylinder_triangles) and cut into parts of <= max_tris triangles that share the cylinder's bounding box (kind 1:
    culling only).  A <mesh> (OBJ / STL, load_mesh) or a <sphere> (hp2.icosphere_triangles) is ONE part of any size with obb None:
    the scene makes it a mesh object (RayScene mesh_templates), its triangles in file order.  link_index counts the links that carry
    a visual, in urdfpy's link order -- the per-link segmentation counter of assets/warp_asset.py:44-70."""
    from .hp2 import box_obb, box_triangles, cylinder_triangles, icosphere_triangles

    tf = model.link_transforms()
    out, link_index = [], 0
    for name in model.body_order():
        l = model.links[name]
        R, p = tf[name]
        had_visual = False
        for v in (l.collisions if use_collision else l.visuals):
            if v.kind == "box":
                t, obb = box_triangles(v.size), box_obb(v.size, R @ v.R, R @ v.p + p)
            elif v.kind == "cylinder":
                t = cylinder_triangles(v.size[0], v.size[1])
                obb = box_obb((2 * v.size[0], 2 * v.size[0], v.size[1]), R @ v.R, R @ v.p + p)
                obb[15] = 1.0
            elif v.kind == "sphere":
                t, obb = icosphere_triangles(v.size[0]), None
            elif v.kind == "mesh":
                t, obb = load_mesh(v.filename, v.size), None
            else:
                continue
            had_visual = True
            t = t.reshape(-1, 3).astype(np.float64)
            t = (R @ (v.R @ t.T + v.p[:, None]) + p[:, None]).T.reshape(-1, 9).astype(np.float32)
            if obb is None:
                out.append((name, link_index, t, None))
                continue
            for i in range(0, len(t), max_tris):
                out.append((name, link_index, t[i:i + max_tris], obb))
        link_index += int(had_visual)
    return out
