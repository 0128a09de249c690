"""Re-author the robot / obstacle descriptions the hot paths need as minimal URDFs.

    python tools/strip_resources.py            (reads $AERIAL_GYM_REFERENCE/resources)

For each source URDF only the physical facts are kept -- link names, inertials, fixed-joint
origins, box geometry of visuals/collisions -- re-serialised from the parsed model (no meshes,
materials or comments).  Output: aerial_gym_simulator_b200/resources/."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from aerial_gym_simulator_b200 import urdf  # noqa: E402

SRC = os.path.join(os.environ.get("AERIAL_GYM_REFERENCE", ""), "resources")
DST = os.path.join(ROOT, "aerial_gym_simulator_b200", "resources")


def mat_to_rpy(R):
    p = -np.arcsin(np.clip(R[2, 0], -1, 1))
    r = np.arctan2(R[2, 1], R[2, 2])
    y = np.arctan2(R[1, 0], R[0, 0])
    return r, p, y


def fmt(v):
    return " ".join(repr(float(x)) for x in v)


def emit(model: urdf.UrdfModel, path):
    out = ['<?xml version="1.0"?>', f'<robot name="{model.name}">']
    for name in model.body_order():
        l = model.links[name]
        out.append(f'  <link name="{name}">')
        out.append("    <inertial>")
        out.append(f'      <origin xyz="{fmt(l.com)}" rpy="{fmt(mat_to_rpy(l.com_R))}"/>')
        out.append(f'      <mass value="{l.mass!r}"/>')
        I = l.inertia
        out.append(f'      <inertia ixx="{float(I[0,0])!r}" ixy="{float(I[0,1])!r}" ixz="{float(I[0,2])!r}" iyy="{float(I[1,1])!r}" iyz="{float(I[1,2])!r}" izz="{float(I[2,2])!r}"/>')
        out.append("    </inertial>")
        for tag, items in (("visual", l.visuals), ("collision", l.collisions)):
            for v in items:
                if v.kind == "box":
                    g = f'<box size="{fmt(v.size)}"/>'
                elif v.kind == "sphere":
                    g = f'<sphere radius="{float(v.size[0])!r}"/>'
                elif v.kind == "cylinder":
                    g = f'<cylinder radius="{float(v.size[0])!r}" length="{float(v.size[1])!r}"/>'
                else:
                    continue  # meshes are not carried
                out.append(f"    <{tag}>")
                out.append(f'      <origin xyz="{fmt(v.p)}" rpy="{fmt(mat_to_rpy(v.R))}"/>')
                out.append(f"      <geometry>{g}</geometry>")
                out.append(f"    </{tag}>")
        out.append("  </link>")
    for j in model.joints:
        out.append(f'  <joint name="{j.name}" type="{j.kind}">')
        out.append(f'    <parent link="{j.parent}"/>')
        out.append(f'    <child link="{j.child}"/>')
        out.append(f'    <origin xyz="{fmt(j.p)}" rpy="{fmt(mat_to_rpy(j.R))}"/>')
        out.append("  </joint>")
    out.append("</robot>")
    os.makedirs(os.path.dirname(path), exist_ok=True)
    open(path, "w").write("\n".join(out) + "\n")


if __name__ == "__main__":
    robots = {"quad/quad.urdf": "robots/quad/quad.urdf", "quad/model.urdf": "robots/quad/model.urdf",
              "octarotor/octarotor.urdf": "robots/octarotor/octarotor.urdf",
              "lmf2/model.urdf": "robots/lmf2/model.urdf", "lmf1/model.urdf": "robots/lmf1/model.urdf",
              "x500/model.urdf": "robots/x500/model.urdf", "magpie/model.urdf": "robots/magpie/model.urdf",
              "tinyprop/tinyprop.urdf": "robots/tinyprop/tinyprop.urdf", "random/random.urdf": "robots/random/random.urdf",
              "BlueROV/rov.urdf": "robots/BlueROV/rov.urdf", "morphy/morphy_stiff.urdf": "robots/morphy/morphy_stiff.urdf"}
    for s, d in robots.items():
        sp = os.path.join(SRC, "robots", s)
        if os.path.exists(sp):
            emit(urdf.parse_urdf(sp), os.path.join(DST, d))
            print("robot", d)
    env = os.path.join(SRC, "models", "environment_assets")
    for sub in ("panels", "objects", "walls", "trees", "thin"):
        for f in sorted(os.listdir(os.path.join(env, sub))):
            if f.endswith(".urdf"):
                emit(urdf.parse_urdf(os.path.join(env, sub, f)), os.path.join(DST, "models", "environment_assets", sub, f))
                print("asset", sub, f)
