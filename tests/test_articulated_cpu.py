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

from . import _articulated_shadow
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
            "motor_p": f(s.motor_p, 3), "motor_torque": f(s.motor_torque)}


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
