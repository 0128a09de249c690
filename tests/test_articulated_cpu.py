"""Articulated multirotors on the CPU (DESIGN.md "Articulated robots"): the merged body table, the articulated-body algorithm of
articulated_core.cuh (host shadow, tests/csrc/articulated_shadow.cu) against the float64 CRBA + RNEA checker
(oracle/articulated_oracle.py), its reductions and physics, and the host layer (EnvManager, PositionSetpointTask) on the CPU stack."""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

from aerial_gym_simulator_b200 import _lib, urdf
from aerial_gym_simulator_b200.hp1 import ArticulationSpec, MultirotorSpec
from oracle import articulated_oracle as AO
from oracle import hp1_oracle as HO

from . import _articulated_shadow
from . import _hp1_common as H
from ._cpu_stack import CpuHp1Engine
from ._cpu_stack_articulated import CpuArticulatedHp1Engine, articulated_cpu_stack
from ._hp1_common import spec_from_registry

MORPHY = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "aerial_gym_simulator_b200", "resources", "robots",
                      "morphy")


def _ptr(a):
    return C.c_void_p(a.ctypes.data)


def table_of(s):
    """AgxArticulation -> the oracle's dict (float64 copies of the float32 values the shadow reads)"""
    B = s.num_bodies
    f = lambda x, *shape: np.array(np.ctypeslib.as_array(x), np.float64).reshape(-1, *shape) if shape else \
        np.array(np.ctypeslib.as_array(x), np.float64)
    return {"num_bodies": B, "parent": np.ctypeslib.as_array(s.parent).copy(), "joint_R": f(s.joint_R, 3, 3), "joint_p": f(s.joint_p, 3),
            "axis": f(s.axis, 3), "mass": f(s.mass), "com": f(s.com, 3), "inertia": f(s.inertia, 3, 3), "stiffness": f(s.stiffness),
            "damping": f(s.damping), "motor_body": np.ctypeslib.as_array(s.motor_body).copy(), "motor_R": f(s.motor_R, 3, 3),
            "motor_p": f(s.motor_p, 3), "motor_torque": f(s.motor_torque), "lower": f(s.lower), "upper": f(s.upper),
            "limited": np.ctypeslib.as_array(s.limited).copy()}


def shadow_dynamics(s, root, q, qd, qs, qds, dt, grav, thrust, F_w, T_w):
    f32 = lambda x: np.ascontiguousarray(x, np.float32)
    root, q, qd, qs, qds, grav, thrust, F_w, T_w = map(f32, (root, q, qd, qs, qds, grav, thrust, F_w, T_w))
    D = s.num_dofs
    a0, qdd = np.zeros(6, np.float32), np.zeros(max(D, 1), np.float32)
    _articulated_shadow.load().shadow_art_dynamics(C.byref(s), _ptr(root), _ptr(q), _ptr(qd), _ptr(qs), _ptr(qds), float(dt), _ptr(grav),
                                                   len(thrust), _ptr(thrust), _ptr(F_w), _ptr(T_w), _ptr(a0), _ptr(qdd))
    return a0.astype(np.float64), qdd[:D].astype(np.float64)


def random_rotation(rng):
    q = rng.normal(size=4)
    return AO.quat_to_matrix(q / np.linalg.norm(q))


def random_bodies(rng, B):
    """a random tree of B bodies: random parents, joint frames, axes, masses and SPD inertias"""
    parent = np.array([-1] + [int(rng.integers(0, i)) for i in range(1, B)])
    jR = np.array([np.eye(3)] + [random_rotation(rng) for _ in range(1, B)])
    jp = np.vstack([np.zeros(3), rng.uniform(-0.2, 0.2, (B - 1, 3))])
    ax = rng.normal(size=(B, 3))
    ax /= np.linalg.norm(ax, axis=1, keepdims=True)
    mass = rng.uniform(0.05, 0.5, B)
    mass[0] = rng.uniform(0.5, 2.0)
    com = rng.uniform(-0.05, 0.05, (B, 3))
    inertia = []
    for i in range(B):
        Rr = random_rotation(rng)
        inertia.append(Rr @ np.diag(rng.uniform(1e-4, 1e-3, 3)) @ Rr.T)
    z = np.zeros(B)
    return urdf.ArticulatedBodies([f"l{i}" for i in range(B)], parent, [""] + [f"j{i}" for i in range(1, B)], [""] + ["revolute"] * (B - 1),
                                  jR, jp, ax, z - 1.0, z + 1.0, np.zeros(B, bool), z.copy(), mass, com, np.array(inertia), {}, {})


def random_art(rng, B, drive=True, M=4):
    bodies = random_bodies(rng, B)
    D = B - 1
    k = rng.uniform(0.0, 5.0, D) if drive else np.zeros(D)
    d = rng.uniform(0.0, 0.05, D) if drive else np.zeros(D)
    mb = rng.integers(0, B, M)
    return ArticulationSpec(bodies, k, d, mb, np.array([random_rotation(rng) for _ in range(M)]), rng.uniform(-0.1, 0.1, (M, 3)),
                            rng.uniform(-0.02, 0.02, M))


def random_root(rng):
    r = np.zeros(13)
    r[0:3] = rng.uniform(-5, 5, 3)
    qq = rng.normal(size=4)
    r[3:7] = qq / np.linalg.norm(qq)
    r[7:13] = rng.uniform(-2, 2, 6)
    return r


def morphy_compliant():
    import aerial_gym_simulator_b200.robots  # noqa: F401
    from aerial_gym_simulator_b200.config.env_config import EmptyEnvCfg
    from aerial_gym_simulator_b200.registry._core import robot_registry
    robot, _ = robot_registry.make_robot("morphy_compliant", "lee_attitude_control", EmptyEnvCfg, "cpu")
    return robot, robot.make_articulation()


# ---- 1. body table ---------------------------------------------------------------------------------------------------------
def test_morphy_compliant_body_table():
    model = urdf.parse_urdf(os.path.join(MORPHY, "morphy_compliant.urdf"))
    b = model.articulation()
    assert b.num_bodies == 9 and b.num_dofs == 8
    assert list(b.parent) == [-1, 0, 1, 0, 3, 0, 5, 0, 7]
    tf = model.link_transforms()
    for arm in range(4):
        sweep, flap = 1 + 2 * arm, 2 + 2 * arm
        assert b.joint_names[sweep] == f"base_link_to_connecting_link_{arm}"
        assert b.joint_names[flap] == f"connecting_link_to_arm_motor_{arm}"
        np.testing.assert_allclose(tf[b.links[sweep]][0] @ b.axis[sweep], [0, 0, -1], atol=1e-12)  # the arm sweeps in plane
        a = tf[b.links[flap]][0] @ b.axis[flap]
        arm_dir = tf[f"motor_{arm}"][1] - tf[b.links[flap]][1]
        assert abs(a[2]) < 1e-12 and abs(a @ arm_dir) < 1e-12  # horizontal, perpendicular to the arm: it flaps
        assert b.limited[sweep] and b.limited[flap] and b.lower[flap] == -0.6 and b.upper[flap] == 0.6
    # merged mass properties at q = 0 = composite_inertia()
    m, com, J = model.composite_inertia()
    R0, P0 = [np.eye(3)], [np.zeros(3)]
    for i in range(1, b.num_bodies):
        R0.append(R0[b.parent[i]] @ b.joint_R[i])
        P0.append(P0[b.parent[i]] + R0[b.parent[i]] @ b.joint_p[i])
    cw = [P0[i] + R0[i] @ b.com[i] for i in range(b.num_bodies)]
    assert abs(b.mass.sum() - m) < 1e-12
    np.testing.assert_allclose(sum(b.mass[i] * cw[i] for i in range(b.num_bodies)) / b.mass.sum(), com, atol=1e-12)
    Jm = sum(R0[i] @ b.inertia[i] @ R0[i].T + b.mass[i] * (float((cw[i] - com) @ (cw[i] - com)) * np.eye(3) - np.outer(cw[i] - com, cw[i] - com))
             for i in range(b.num_bodies))
    np.testing.assert_allclose(Jm, J, atol=1e-12)
    # an all-fixed URDF is one body
    assert urdf.parse_urdf(os.path.join(MORPHY, "morphy_stiff.urdf")).articulation().num_bodies == 1


def _urdf(tmp_path, joints, n_links=None, axis="1 0 0", mass=1.0):
    J = lambda i: 1e-3 if (mass or not i) else 0.0
    links = "".join(f'<link name="l{i}"><inertial><mass value="{mass if i else 1.0}"/><origin xyz="0 0 0.1"/>'
                    f'<inertia ixx="{J(i)}" iyy="{J(i)}" izz="{J(i)}" ixy="0" ixz="0" iyz="0"/></inertial></link>'
                    for i in range((n_links or len(joints)) + 1))
    js = "".join(f'<joint name="j{i + 1}" type="{kind}"><parent link="l{i}"/><child link="l{i + 1}"/><origin xyz="0 0 0.1"/>'
                 f'<axis xyz="{axis}"/></joint>' for i, kind in enumerate(joints))
    p = tmp_path / "t.urdf"
    p.write_text(f'<robot name="t">{links}{js}</robot>')
    return urdf.parse_urdf(str(p))


@pytest.mark.parametrize("kind", ["prismatic", "planar", "floating"])
def test_unsupported_joint_kinds_raise(tmp_path, kind):
    m = _urdf(tmp_path, ["revolute", kind])  # parse_urdf itself stays permissive
    with pytest.raises(ValueError, match=f"joint 'j2' is {kind}"):
        m.articulation()


def test_more_than_sixteen_bodies_raise(tmp_path):
    assert _urdf(tmp_path, ["revolute"] * 15).articulation().num_bodies == 16
    with pytest.raises(ValueError, match="at most 16"):
        _urdf(tmp_path, ["revolute"] * 16).articulation()


def test_zero_axis_raises(tmp_path):
    with pytest.raises(ValueError, match="zero <axis>"):
        _urdf(tmp_path, ["revolute"], axis="0 0 0").articulation()


def test_massless_undriven_subtree_raises(tmp_path):
    b = _urdf(tmp_path, ["revolute"], mass=0.0).articulation()
    mk = lambda k, d: ArticulationSpec(b, k, d, [0] * 4, np.tile(np.eye(3), (4, 1, 1)), np.zeros((4, 3)), np.zeros(4))
    with pytest.raises(ValueError, match="no inertia about the axis"):
        mk(0.0, 0.0)
    mk(1.0, 0.0)  # a drive makes the pivot non-zero
    mk(0.0, 0.1)


# ---- 2. ABA against CRBA -----------------------------------------------------------------------------------------------------
RTOL = 2e-4  # float32 ABA vs float64 CRBA, relative to the largest entry of (a0, qdd): measured worst case ~2e-5 on these draws


def _check_against_oracle(spec, rng, scale_q=1.0):
    s = spec.to_struct()
    D = s.num_dofs
    root = random_root(rng)
    q, qd = rng.uniform(-scale_q, scale_q, D), rng.uniform(-3, 3, D)
    qs, qds = rng.uniform(-1, 1, D), rng.uniform(-1, 1, D)
    thrust = rng.uniform(0, 2, len(spec.motor_body))
    F, T = rng.uniform(-1, 1, 3), rng.uniform(-0.05, 0.05, 3)
    grav, dt = np.array([0.0, 0.0, -9.81]), 0.01
    a_s, qdd_s = shadow_dynamics(s, root, q, qd, qs, qds, dt, grav, thrust, F, T)
    a_o, qdd_o = AO.dynamics(table_of(s), np.float32(root).astype(np.float64), np.float32(q).astype(np.float64),
                             np.float32(qd).astype(np.float64), np.float32(qs).astype(np.float64), np.float32(qds).astype(np.float64),
                             dt, grav, np.float32(thrust).astype(np.float64), np.float32(F).astype(np.float64), np.float32(T).astype(np.float64))
    ref = np.concatenate([a_o, qdd_o])
    err = np.abs(np.concatenate([a_s, qdd_s]) - ref).max() / np.abs(ref).max()
    assert err < RTOL, err


def test_aba_matches_crba_on_morphy_compliant():
    _, art = morphy_compliant()
    rng = np.random.default_rng(1)
    for _ in range(50):
        _check_against_oracle(art, rng, scale_q=0.6)


@pytest.mark.parametrize("drive", [True, False])
def test_aba_matches_crba_on_random_trees(drive):
    rng = np.random.default_rng(7 + drive)
    for trial in range(60):
        B = int(rng.integers(1, 17))
        _check_against_oracle(random_art(rng, B, drive=drive), rng)


# ---- 3. zero-DOF reduction ---------------------------------------------------------------------------------------------------
def _stiff_pair(n=64, seed=0, **over):
    spec = spec_from_registry("morphy_stiff", "lee_attitude_control")
    for k, v in over.items():
        setattr(spec, k, v)
    model = urdf.parse_urdf(os.path.join(MORPHY, "morphy_stiff.urdf"))
    b = model.articulation()
    order = model.body_order()
    mR, mp = zip(*[b.link_in_body[order[i]] for i in (3, 6, 9, 12)])
    art = ArticulationSpec(b, [], [], [0] * 4, np.array(mR), np.array(mp), -spec.thrust_to_torque_ratio * spec.motor_directions)
    hp1 = CpuHp1Engine(spec, n, per_env_params="all")
    arte = CpuArticulatedHp1Engine(spec, n, per_env_params="all", articulation=art)
    return spec, hp1, arte


def _random_start(engines, n, rng, v=0.5, w=0.8):
    root = torch.zeros(n, 13)
    root[:, 0:3] = torch.from_numpy(rng.uniform(-1, 1, (n, 3))).float()
    qq = torch.from_numpy(rng.normal(size=(n, 4))).float()
    qq[:, 0:2] *= 0.1
    root[:, 3:7] = qq / qq.norm(dim=1, keepdim=True)
    root[:, 7:10] = torch.from_numpy(rng.uniform(-v, v, (n, 3))).float()
    root[:, 10:13] = torch.from_numpy(rng.uniform(-w, w, (n, 3))).float()
    thrust = torch.from_numpy(rng.uniform(0.5, 1.0, (n, 4))).float()
    for e in engines:
        e.root_state.copy_(root)
        e.motor_thrust.copy_(thrust)


def test_zero_dof_tree_reduces_to_hp1_integrate():
    """morphy_stiff pushed through the articulated path (one body, no DOF) against the HP1 shadow, 100 sub-steps, with the
    damping factors and both velocity caps active (caps set just below the start speeds)"""
    n = 64
    spec, hp1, arte = _stiff_pair(n, max_linear_velocity=0.6, max_angular_velocity=0.9, linear_damping=0.5, angular_damping=0.5)
    rng = np.random.default_rng(3)
    _random_start((hp1, arte), n, rng)
    act = torch.from_numpy(rng.uniform(-0.3, 0.3, (n, 4))).float()
    capped = False
    for _ in range(100):
        hp1.physics_step(act, physics_steps=1)
        arte.physics_step(act, physics_steps=1)
        capped |= bool((hp1.root_state[:, 7:10].norm(dim=1) > 0.599).any())
    assert capped
    d = (arte.root_state - hp1.root_state).abs().max().item()
    assert d < 2e-5, d  # float32 rounding: the two forms of the same update round differently
    assert (arte.motor_thrust - hp1.motor_thrust).abs().max().item() < 2e-5


# ---- 4. stiff limit ----------------------------------------------------------------------------------------------------------
def test_stiff_joints_track_morphy_stiff():
    """k = 1e4 N m / rad on every joint: the arms deflect by ~4e-6 rad under hover thrust, so morphy_compliant follows morphy_stiff's
    HP1 trajectory over 1 s of random attitude commands.  Tolerance: 1e-3 m / 1e-3 in the quaternion -- the remaining differences
    are the micro-radian deflections (which tilt the thrust by as much) integrated over 100 sub-steps, plus float32 rounding."""
    n = 32
    robot, art = morphy_compliant()
    art.stiffness[:] = 1e4
    spec = spec_from_registry("morphy_stiff", "lee_attitude_control")
    hp1 = CpuHp1Engine(spec, n, per_env_params="all")
    arte = CpuArticulatedHp1Engine(spec, n, per_env_params="all", articulation=art)
    rng = np.random.default_rng(5)
    _random_start((hp1, arte), n, rng, v=0.2, w=0.2)
    for _ in range(10):
        act = torch.from_numpy(rng.uniform(-0.3, 0.3, (n, 4))).float()
        hp1.physics_step(act, physics_steps=10)
        arte.physics_step(act, physics_steps=10)
    assert (arte.root_state[:, 0:3] - hp1.root_state[:, 0:3]).abs().max().item() < 1e-3
    assert (arte.root_state[:, 3:7] - hp1.root_state[:, 3:7]).abs().max().item() < 1e-3
    assert arte.dof_state[..., 0].abs().max().item() < 1e-4


# ---- 5. physics ----------------------------------------------------------------------------------------------------------------
def _single_joint_engine(tmp_path, n, k=0.0, d=0.0, L=0.5, base_mass=1e6, grav=(0.0, 0.0, -9.81), dt=0.001, limit=None):
    lim = f'<limit lower="{limit[0]}" upper="{limit[1]}"/>' if limit else ""
    text = (f'<robot name="p"><link name="base"><inertial><mass value="{base_mass}"/>'
            f'<inertia ixx="{base_mass}" iyy="{base_mass}" izz="{base_mass}" ixy="0" ixz="0" iyz="0"/></inertial></link>'
            f'<link name="bob"><inertial><origin xyz="0 0 {-L}"/><mass value="0.1"/>'
            f'<inertia ixx="0" iyy="0" izz="0" ixy="0" ixz="0" iyz="0"/></inertial></link>'
            f'<joint name="hinge" type="revolute"><parent link="base"/><child link="bob"/><axis xyz="1 0 0"/>{lim}</joint></robot>')
    p = tmp_path / "p.urdf"
    p.write_text(text)
    b = urdf.parse_urdf(str(p)).articulation()
    art = ArticulationSpec(b, k, d, [0] * 4, np.tile(np.eye(3), (4, 1, 1)), np.zeros((4, 3)), np.zeros(4))
    spec = MultirotorSpec(controller=_lib.CTRL_NONE, dt=dt, gravity=grav, mass=base_mass, inertia=np.eye(3) * base_mass,
                          linear_damping=0.0, angular_damping=0.0)
    eng = CpuArticulatedHp1Engine(spec, n, per_env_params="all", articulation=art)
    # the base is held against gravity (otherwise base and bob fall together and nothing swings): a body-frame force on the base,
    # through the disturbance input, equal to the total weight
    support = torch.zeros(n, 6)
    support[:, 0:3] = -torch.tensor(grav, dtype=torch.float64) * (base_mass + 0.1)
    eng.support = support.float()
    return eng, torch.zeros(n, 4)


def test_pendulum_small_angle_period(tmp_path):
    L, g = 0.5, 9.81
    eng, act = _single_joint_engine(tmp_path, 1, L=L)
    eng.dof_state[0, 0, 0] = 0.02
    qs, steps = [], 4000
    for _ in range(steps):
        eng.physics_step(act, disturbance=eng.support, physics_steps=1)
        qs.append(float(eng.dof_state[0, 0, 0]))
    qs = np.array(qs)
    up = np.nonzero((qs[:-1] < 0) & (qs[1:] >= 0))[0]
    crossings = up + (-qs[up]) / (qs[up + 1] - qs[up])  # linear interpolation of the upward zero crossings
    T = np.diff(crossings).mean() * 0.001
    assert abs(T / (2 * math.pi * math.sqrt(L / g)) - 1) < 0.01, T


def test_free_tree_momentum_drift_falls_with_dt():
    """gravity off, no drive, no motors: the drift of linear momentum and of angular momentum about the COM over 0.2 s falls at
    least linearly when dt is halved"""
    rng = np.random.default_rng(11)
    spec_a = random_art(rng, 6, drive=False)
    spec_a.motor_body[:] = 0
    tab = table_of(spec_a.to_struct())
    root0, q0, qd0 = random_root(rng), rng.uniform(-1, 1, 5), rng.uniform(-2, 2, 5)
    drifts = []
    for dt in (0.002, 0.001):
        ms = MultirotorSpec(controller=_lib.CTRL_NONE, dt=dt, gravity=(0.0, 0.0, 0.0), mass=float(spec_a.bodies.mass[0]),
                            linear_damping=0.0, angular_damping=0.0, max_linear_velocity=1e6, max_angular_velocity=1e6)
        eng = CpuArticulatedHp1Engine(ms, 1, per_env_params="all", articulation=spec_a)
        eng.root_state[0] = torch.tensor(root0, dtype=torch.float32)
        eng.dof_state[0, :, 0] = torch.tensor(q0, dtype=torch.float32)
        eng.dof_state[0, :, 1] = torch.tensor(qd0, dtype=torch.float32)
        mom = lambda: AO.momentum(tab, eng.root_state[0].double().numpy(), eng.dof_state[0, :, 0].double().numpy(),
                                  eng.dof_state[0, :, 1].double().numpy())
        p0, L0 = mom()
        eng.physics_step(torch.zeros(1, 4), physics_steps=int(round(0.2 / dt)))
        p1, L1 = mom()
        drifts.append((np.linalg.norm(p1 - p0), np.linalg.norm(L1 - L0)))
    (p_a, l_a), (p_b, l_b) = drifts
    assert p_b <= 0.5 * p_a * 1.05 + 1e-6 and l_b <= 0.5 * l_a * 1.05 + 1e-7, drifts


def test_implicit_drive_is_stable_and_settles_at_tau_over_k(tmp_path):
    """w dt = 35 (the explicit drive would blow up): the implicit one stays bounded and settles where the spring holds gravity"""
    L, m, g, dt = 0.5, 0.1, 9.81, 0.01
    inertia = m * L * L
    k = (35.0 / dt) ** 2 * inertia
    eng, act = _single_joint_engine(tmp_path, 1, k=k, d=0.0, L=L, grav=(0.0, -g, 0.0), dt=dt)  # gravity along -y: torque about x
    eng.dof_state[0, 0, 0] = 0.3
    peak = 0.0
    for _ in range(300):
        eng.physics_step(act, disturbance=eng.support, physics_steps=1)
        peak = max(peak, abs(float(eng.dof_state[0, 0, 0])))
    assert peak <= 0.3 + 1e-6
    tau = -m * g * L  # bob at (0, 0, -L): gravity -g y gives torque (r x F).x = -L * m g ... about +x: -m g L
    np.testing.assert_allclose(float(eng.dof_state[0, 0, 0]), tau / k, rtol=1e-3)


def test_limit_projection(tmp_path):
    eng, act = _single_joint_engine(tmp_path, 2, L=0.5, grav=(0.0, -9.81, 0.0), limit=(-0.2, 0.3), dt=0.005)
    eng.dof_state[:, 0, 1] = torch.tensor([5.0, -5.0])
    for _ in range(50):
        eng.physics_step(act, disturbance=eng.support, physics_steps=1)
        q, qd = eng.dof_state[:, 0, 0], eng.dof_state[:, 0, 1]
        assert (q >= -0.2).all() and (q <= 0.3).all()
        assert not ((q == 0.3) & (qd > 0)).any() and not ((q == -0.2) & (qd < 0)).any()
    assert float(eng.dof_state[1, 0, 0]) == pytest.approx(-0.2)  # gravity holds it against the lower stop


def _hover_env(n=16, steps=300):
    from aerial_gym_simulator_b200.env_manager.env_manager import EnvManager
    env = EnvManager("base_sim", "empty_env", "morphy_compliant", "lee_attitude_control", "cpu", num_envs=n)
    env.spec.enable_disturbance = False
    env.reset()
    gtd = env.global_tensor_dict
    gtd["dof_state_tensor"].zero_()
    st = gtd["robot_state_tensor"]
    st[:, 3:13] = 0.0
    st[:, 6] = 1.0
    for _ in range(steps):
        env.step(torch.zeros(n, 4))
    return env


def hover_check(env):
    """flap deflection at hover: the thrust's moment about the flap hinge less the motor's own weight's, over k.  (The motor mass
    0.01625 kg sits at the arm's end, so with f = 0.71 N the weight takes 22 % off f * 0.07 / k.)"""
    gtd = env.global_tensor_dict
    eng = env.engine
    f = eng.motor_thrust.double()
    k = float(env.robot_cfg.joint_config.stiffness)
    expect = -(f - 0.01625 * 9.81) * 0.07 / k
    flap = gtd["dof_state_tensor"][:, 1::2, 0].double()
    assert (flap - expect).abs().max().item() <= 0.05 * expect.abs().min().item(), (flap, expect)
    assert gtd["dof_state_tensor"][..., 1].abs().max().item() < 1e-2


def test_hover_flap_deflection():
    with articulated_cpu_stack():
        hover_check(_hover_env())


# ---- 6. host layer -----------------------------------------------------------------------------------------------------------
def _env(robot="morphy_compliant", n=8, **args):
    from aerial_gym_simulator_b200.env_manager.env_manager import EnvManager
    return EnvManager("base_sim", "empty_env", robot, "lee_attitude_control", "cpu", num_envs=n, args=args or None)


def test_gtd_keys_shapes_and_reset_draws():
    with articulated_cpu_stack():
        env = _env(n=64)
        gtd = env.global_tensor_dict
        assert gtd["dof_state_tensor"].shape == (64, 8, 2)
        assert gtd["dof_position_setpoint_tensor"].shape == (64, 8) and gtd["dof_velocity_setpoint_tensor"].shape == (64, 8)
        assert env.IGE_env.sim_has_dof is True
        gtd["dof_position_setpoint_tensor"].fill_(0.25)
        gtd["dof_velocity_setpoint_tensor"].fill_(-0.5)
        env.reset()
        q = gtd["dof_state_tensor"]
        assert (q[..., 0].abs() <= 0.1).all() and q[..., 0].std() > 0.03 and (q[..., 1] == 0).all()
        assert (gtd["dof_position_setpoint_tensor"] == 0.25).all() and (gtd["dof_velocity_setpoint_tensor"] == -0.5).all()
        before = q.clone()
        env.reset_idx(torch.tensor([3]))
        changed = (q != before).any(dim=(1, 2))
        assert changed[3] and not changed[torch.arange(64) != 3].any()
        for _ in range(5):
            env.step(torch.zeros(64, 4))
        assert (gtd["dof_position_setpoint_tensor"] == 0.25).all()


def test_existing_robots_unchanged():
    """no new GTD keys, and the reset draws of the robot (torch order) are those of the parent: the joint draw comes after them"""
    with articulated_cpu_stack():
        torch.manual_seed(0)
        env = _env("morphy_stiff", 16, reset_rng="torch")
        new = ("dof_state_tensor", "dof_position_setpoint_tensor", "dof_velocity_setpoint_tensor")
        assert not any(k in env.global_tensor_dict for k in new) and env.IGE_env.sim_has_dof is False
        env.reset()
        stiff = env.global_tensor_dict["robot_state_tensor"].clone()
        torch.manual_seed(0)
        env2 = _env("morphy_compliant", 16, reset_rng="torch")
        env2.reset()
        assert torch.equal(env2.global_tensor_dict["robot_state_tensor"], stiff)


def test_unsupported_combinations_raise():
    with articulated_cpu_stack():
        with pytest.raises(ValueError, match="impulse to the base alone"):
            _env(contact="rigid")
        with pytest.raises(NotImplementedError, match="fused task step"):
            _env(host_io=True)
    from aerial_gym_simulator_b200.config import robot_config as rc
    from aerial_gym_simulator_b200.registry._core import robot_registry

    class WithImu(rc.MorphyCompliantCfg):
        class sensor_config(rc.MorphyCompliantCfg.sensor_config):
            enable_imu = True

    class RootLink(rc.MorphyCompliantCfg):
        class control_allocator_config(rc.MorphyCompliantCfg.control_allocator_config):
            force_application_level = "root_link"

    from aerial_gym_simulator_b200.robots import ArticulatedMultirotor
    robot_registry.register("_test_morphy_imu", ArticulatedMultirotor, WithImu)
    robot_registry.register("_test_morphy_root", ArticulatedMultirotor, RootLink)
    with articulated_cpu_stack():
        with pytest.raises(ValueError, match="joint reaction forces"):
            _env("_test_morphy_imu")
        with pytest.raises(ValueError, match="root_link"):
            _env("_test_morphy_root")


def test_position_task_runs_unfused(monkeypatch):
    from aerial_gym_simulator_b200.registry._core import task_registry
    import aerial_gym_simulator_b200.task  # noqa: F401
    cfg = task_registry.get_task_config("position_setpoint_task")
    monkeypatch.setattr(cfg, "robot_name", "morphy_compliant")
    monkeypatch.setattr(cfg, "device", "cpu")
    with articulated_cpu_stack():
        task = task_registry.make_task("position_setpoint_task", seed=1, num_envs=16, headless=True)
        assert task._unfused
        task.reset()
        g = torch.Generator().manual_seed(0)
        for _ in range(20):
            obs, rew, term, trunc, _ = task.step(torch.rand(16, 4, generator=g) * 2 - 1)
        assert torch.isfinite(obs["observations"]).all() and torch.isfinite(rew).all()
        q = task.sim_env.global_tensor_dict["dof_state_tensor"][..., 0]
        assert (q.abs() <= 0.6 + 1e-6).all()


# ---- 7. one whole sub-step against the float64 reference ---------------------------------------------------------------------
# Tolerance of a sub-step's state against AO.substep, derived from the ABA's bar: the float32 ABA is within RTOL of
# amax = max |(a0, qdd)| of the env (section 2), and the sub-step carries that error through one dt into the velocities (base
# v, w and qd) and through dt^2 into the positions (base x and quaternion, q); on top comes the float32 rounding of the update
# itself, at most ULPS ulps of the magnitude of the quantity (its value before or after the sub-step, whichever is larger).
# Measured worst case over tests/test_zz_articulated_oracle_gpu.py, as a fraction of this tolerance: 0.56 on the host shadow
# (qd), 0.34 on the H100 (qd; H100 80GB HBM3).
EPS32 = 2.0 ** -23
ULPS = 8


def shaped_art(rng, B, shape="random", M=4, drive=True, motors="random"):
    """random_art with the tree's shape and the motors' bodies chosen: shape "chain" (depth B - 1), "star" (every joint on the
    base) or "random"; motors "base" (all on body 0), "leaves" (round robin over the bodies without children), "cluster" (all but
    one on the last body) or "random\""""
    art = random_art(rng, B, drive=drive, M=M)
    b = art.bodies
    if shape == "chain":
        b.parent[1:] = np.arange(B - 1)
    elif shape == "star":
        b.parent[1:] = 0
    leaves = [i for i in range(B) if i not in set(b.parent[1:].tolist())]
    if motors == "base":
        art.motor_body[:] = 0
    elif motors == "leaves":
        art.motor_body[:] = [leaves[k % len(leaves)] for k in range(M)]
    elif motors == "cluster":
        art.motor_body[:] = B - 1
        art.motor_body[0] = 0
    return art


def substep_inputs(spec, art, N, seed):
    """seeded inputs of one sub-step (CPU float32 tensors): root, actions, motor constants and gains of _hp1_common.random_inputs,
    joint state within +-0.8 rad and +-3 rad/s (inside the limits of a limited joint), drive targets, a body-frame disturbance"""
    root, actions, params = H.random_inputs(spec, N, seed)
    rng = np.random.default_rng(seed)
    b, D = art.bodies, art.num_dofs
    lo = np.where(b.limited[1:], b.lower[1:], -0.8)
    hi = np.where(b.limited[1:], b.upper[1:], 0.8)
    q = lo + (hi - lo) * rng.uniform(0.0, 1.0, (N, D))
    f32 = lambda a: torch.tensor(np.asarray(a, np.float32))
    return {"root": root, "actions": actions, "params": params, "dof": f32(np.stack([q, rng.uniform(-3, 3, (N, D))], -1)),
            "qs": f32(rng.uniform(-0.5, 0.5, (N, D))), "qds": f32(rng.uniform(-1, 1, (N, D))),
            "dist": f32(rng.uniform(-0.3, 0.3, (N, 6)) * [1, 1, 1, 0.01, 0.01, 0.01])}


def load_inputs(eng, inp):
    H.load_engine_state(eng, inp["root"], inp["params"])
    dev = eng.root_state.device
    eng.dof_state.copy_(inp["dof"].to(dev))
    eng.dof_position_setpoint.copy_(inp["qs"].to(dev))
    eng.dof_velocity_setpoint.copy_(inp["qds"].to(dev))


def oracle_state(eng, spec, inp, idx):
    """hp1_oracle's model and float64 state of envs idx: what the kernel reads -- the per-env arrays the engine holds, the
    config's float32 constants for the parameters it does not (per_env_params="auto")"""
    model = H.oracle_model_from_spec(spec)
    n, M = len(idx), spec.num_motors
    st = HO.make_state(model, n, torch.float64)
    st.root, st.thrust = inp["root"][idx].double(), inp["params"]["thrust"][idx].double()
    for k in ("tau_inc", "tau_dec", "k_thrust", "K_pos", "K_vel", "K_rot", "K_angvel"):
        if getattr(eng, k) is not None:
            setattr(st, k, inp["params"][k][idx].double())
        else:
            c = getattr(eng.cfg, k)
            c = [float(c)] * M if k in ("tau_inc", "tau_dec", "k_thrust") else [float(v) for v in c]
            setattr(st, k, torch.tensor(c, dtype=torch.float64).expand(n, -1).clone())
    return model, st


def reference_substep(eng, spec, art, inp, idx):
    """AO.substep on envs idx -> (reference dict, well-conditioned mask [len(idx)])"""
    model, st = oracle_state(eng, spec, inp, idx)
    ok = H.well_conditioned(model, st, inp["actions"][idx].double()).numpy()
    dof = inp["dof"][idx].double().numpy()
    ref = AO.substep(model, table_of(eng.art), st, dof[..., 0], dof[..., 1], inp["qs"][idx].double().numpy(),
                     inp["qds"][idx].double().numpy(), inp["actions"][idx].double(), inp["dist"][idx].double())
    return ref, ok


def _record(worst, what, err, tol):
    r = float((err / tol).max()) if err.size else 0.0
    if worst is not None:
        worst[what] = max(worst.get(what, (0.0, 0.0)), (r, float(err.max()) if err.size else 0.0))
    return r


LIMIT_BAND = 1e-5  # a reference q' this close to a limit may round to either side of it: the projection may go either way


def near_limit(tab, ref):
    """bool [n]: envs with a limited joint whose unprojected reference q' lies within LIMIT_BAND of one of its limits"""
    D = int(tab["num_bodies"]) - 1
    lim = tab["limited"][1:D + 1].astype(bool)
    lo, hi, qf = tab["lower"][1:D + 1], tab["upper"][1:D + 1], ref["q_free"]
    return (lim & ((np.abs(qf - lo) < LIMIT_BAND) | (np.abs(qf - hi) < LIMIT_BAND))).any(1)


def check_substep(eng, spec, inp, ref, ok, idx, worst=None):
    """the engine's state after one sub-step (envs idx) against the reference, with the tolerance above.  Envs that fail
    _hp1_common.well_conditioned, and those near_limit, are only checked for finite values.  worst: a dict that collects
    (worst err / tol, worst |err|) per quantity.  -> the number of envs left out for a joint near a limit"""
    dt = spec.dt
    got = lambda t: t.detach().cpu().double().numpy()[idx]
    root, dof, thrust = got(eng.root_state), got(eng.dof_state), got(eng.motor_thrust)
    for t in (root, dof, thrust):
        assert np.isfinite(t).all()
    near = near_limit(table_of(eng.art), ref)
    keep = ok & ~near
    amax = np.abs(np.concatenate([ref["a0"], ref["qdd"]], 1)).max(1)[keep][:, None]
    r_in, dof_in = inp["root"][idx].double().numpy()[keep], inp["dof"][idx].double().numpy()[keep]
    r_ref = ref["root"][keep]
    mag = lambda *a: np.max([np.abs(x).max(-1, keepdims=True) for x in a], 0)
    checks = {
        "x": (root[keep, 0:3], r_ref[:, 0:3], mag(r_ref[:, 0:3], r_in[:, 0:3]) + dt * mag(r_ref[:, 7:10]), 2),
        "quat": (root[keep, 3:7], r_ref[:, 3:7], 1.0 + dt * mag(r_ref[:, 10:13]), 2),
        "v": (root[keep, 7:10], r_ref[:, 7:10], mag(r_ref[:, 7:10], r_in[:, 7:10]), 1),
        "w": (root[keep, 10:13], r_ref[:, 10:13], mag(r_ref[:, 10:13], r_in[:, 10:13]), 1),
        "q": (dof[keep, :, 0], ref["q"][keep], np.maximum(np.abs(ref["q"][keep]), np.abs(dof_in[..., 0])) + dt * np.abs(ref["qd"][keep]), 2),
        "qd": (dof[keep, :, 1], ref["qd"][keep], np.maximum(np.abs(ref["qd"][keep]), np.abs(dof_in[..., 1])), 1),
    }
    for what, (g, r, m, p) in checks.items():
        err = np.abs(g - r)
        tol = ULPS * EPS32 * m + dt ** p * RTOL * amax
        bad = ~(err <= tol)
        assert not bad.any(), f"{what}: {bad.sum()}/{bad.size} outside tol, worst err/tol {(err / tol).max():.3g} at env " \
                              f"{np.asarray(idx)[keep][np.argwhere(bad)[0][0]]}"
        _record(worst, what, err, tol)
    fs = max(1.0, float(np.abs(ref["thrust"][ok]).max(initial=0.0)))
    H.assert_close(thrust[ok], ref["thrust"][ok], "motor_thrust", scale=fs)
    _record(worst, "thrust", np.abs(thrust[ok] - ref["thrust"][ok]), H.RTOL * np.maximum(np.abs(ref["thrust"][ok]), fs))
    check_derived(eng, ref["derived"], idx, ok, worst)
    return int(near.sum())


def check_derived(eng, d, idx, ok, worst=None):
    """the five derived outputs against update_states in float64 (_hp1_common's scales)"""
    for k, scale in (("euler", math.pi), ("vehicle_orientation", 1.0), ("vehicle_linvel", None), ("body_linvel", None),
                     ("body_angvel", None)):
        g = getattr(eng, k).detach().cpu().double().numpy()[idx]
        assert np.isfinite(g).all(), k
        g, r = g[ok], d[k][ok]
        s = scale if scale is not None else max(float(np.abs(r).max(initial=0.0)), 1e-30)
        H.assert_close(g, r, k, scale=s)
        _record(worst, k, np.abs(g - r), H.RTOL * np.maximum(np.abs(r), s))


def test_substep_reference_reduces_to_hp1_physics_step():
    """One body, its COM at the base origin, the same mass and inertia as the HP1 model, gyroscopic term on: there the ABA's
    floating base is the rigid body of DESIGN section 3, and AO.substep must be hp1_oracle.physics_step (float64 both, drag,
    disturbance, damping and both caps active).  Measured residual: 2.8e-15 absolute, 1.3e-15 relative to the env's state."""
    n = 256
    spec = H.spec_for("quad_attitude")
    spec.drag_lin1, spec.drag_lin2, spec.drag_ang1, spec.drag_ang2 = (0.1, 0.1, 0.2), (0.05, 0.05, 0.1), (1e-3,) * 3, (5e-4,) * 3
    spec.linear_damping, spec.angular_damping, spec.max_linear_velocity, spec.max_angular_velocity = 0.3, 0.4, 1.5, 2.5
    model = H.oracle_model_from_spec(spec)
    assert model.gyroscopic and not model.com.any()
    # the table in float64 (table_of would round it to the float32 struct): body 0 = the HP1 rigid body, the motors its links
    z1 = np.zeros(1)
    tab = {"num_bodies": 1, "parent": np.array([-1]), "joint_R": np.eye(3)[None], "joint_p": np.zeros((1, 3)), "axis": np.zeros((1, 3)),
           "mass": np.array([model.mass]), "com": np.zeros((1, 3)), "inertia": model.inertia[None], "stiffness": z1, "damping": z1,
           "motor_body": np.zeros(4, int), "motor_R": model.link_R, "motor_p": model.link_r,
           "motor_torque": -model.thrust_to_torque_ratio * model.motor_directions, "lower": z1, "upper": z1, "limited": z1}
    root, actions, params = H.random_inputs(spec, n, 17)
    st = H.load_oracle_state(model, root.double(), {k: v.double() for k, v in params.items()}, n)
    st.root[:, 3:7] /= st.root[:, 3:7].norm(dim=1, keepdim=True)  # unit in float64: the two sides rotate by different formulas
    st.root[:, 7:13] *= 1.5  # most envs start above a cap
    dist = torch.rand(n, 6, dtype=torch.float64, generator=torch.Generator().manual_seed(2)) - 0.5
    z = np.zeros((n, 0))
    ref = AO.substep(model, tab, st.clone(), z, z, z, z, actions.double(), dist)
    st1 = st.clone()
    HO.physics_step(model, st1, actions.double(), dist)
    scale = st1.root.abs().max(dim=1, keepdim=True).values.numpy()
    assert np.abs(ref["root"] - st1.root.numpy()).max() <= 1e-9 * scale.max()
    assert (np.abs(ref["root"] - st1.root.numpy()) / scale).max() < 1e-12
    np.testing.assert_allclose(ref["thrust"], st1.thrust.numpy(), rtol=1e-12, atol=0)
    for k, v in st1.derived.items():
        np.testing.assert_array_equal(ref["derived"][k], v.numpy())
    capped = (st.root[:, 7:10].norm(dim=1) > 1.5) & (torch.from_numpy(ref["root"][:, 7:10]).norm(dim=1) > 1.5 - 1e-9)
    assert capped.any()


@pytest.mark.parametrize("M", [4, 8])
def test_shadow_substep_matches_reference_on_random_trees(M):
    """shadow_art_step (one sub-step) against AO.substep on random trees of 1-16 bodies, with the tolerance of section 7"""
    rng = np.random.default_rng(40 + M)
    spec = H.spec_for("quad_attitude" if M == 4 else "octa_velocity")
    worst = {}
    for trial in range(16):
        B = trial + 1
        art = shaped_art(rng, B, M=M, drive=bool(trial % 2))
        n = 24
        eng = CpuArticulatedHp1Engine(spec, n, per_env_params="all", articulation=art)
        inp = substep_inputs(spec, art, n, 100 + trial)
        load_inputs(eng, inp)
        eng.physics_step(inp["actions"], disturbance=inp["dist"], physics_steps=1)
        idx = np.arange(n)
        ref, ok = reference_substep(eng, spec, art, inp, idx)
        assert ok.mean() > 0.8
        check_substep(eng, spec, inp, ref, ok, idx, worst)
    print({k: f"{v[0]:.2f} ({v[1]:.1e})" for k, v in worst.items()})
