"""Prismatic joints of articulated robots on the CPU (DESIGN.md "Articulated robots", "Prismatic joints"): the URDF body table and
the host checks, the float64 oracle's own physics with sliders (oracle/articulated_prismatic_oracle.py), art_env_step with
PRISM (host shadow, tests/csrc/articulated_prismatic_shadow.cu) against it on random trees mixing revolute, continuous and prismatic joints,
bit identity with the other steps on revolute-only trees, the stiff limit of the shipped sliding-payload quadrotor, the host layer
on the CPU stack, the C ABI's checks and the new kernels' machine code."""
import ctypes as C
import dataclasses
import math
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from aerial_gym_simulator_b200 import _build, _lib, urdf
from aerial_gym_simulator_b200.hp1 import ArticulationSpec, MultirotorSpec, build_config
from oracle import articulated_body_state_oracle as BO
from oracle import articulated_effort_oracle as EO
from oracle import articulated_imu_oracle as IO
from oracle import articulated_joint_force_oracle as JO
from oracle import articulated_oracle as AO
from oracle import articulated_prismatic_oracle as PO

from . import _articulated_prismatic_shadow
from . import _hp1_common as H
from ._cpu_stack import CpuHp1Engine
from ._cpu_stack_articulated_prismatic import CpuPrismaticHp1Engine, prismatic_cpu_stack
from ._hp1_common import spec_from_registry
from .test_articulated_cpu import _random_start, check_substep, load_inputs, oracle_state, random_bodies, random_root, \
    random_rotation, substep_inputs, table_of
from .test_articulated_imu_cpu import _depth, _limit_crossing, imu_tolerance
from .test_articulated_joint_force_cpu import check_dof_force_identity, jf_tolerance

EPS = float(np.finfo(np.float32).eps)
QUAD = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "aerial_gym_simulator_b200", "resources", "robots",
                    "quad")
ROBOT = "base_quadrotor_with_sliding_payload"


def ptable(s, mask):
    """table_of(s) with the joint kinds of prismatic_mask `mask`"""
    t = table_of(s)
    t["prismatic"] = np.array([bool((mask >> i) & 1) for i in range(s.num_bodies)])
    return t


def mixed_art(rng, B, M=4, drive=True, effort=False):
    """a random tree of B bodies whose joints are revolute (half of them limited to +-0.6 rad), continuous or prismatic (limited
    to a random range of a few cm either side of 0); drives on or off; with `effort`, about a third of the DOFs in effort mode, some
    with a limit"""
    b = random_bodies(rng, B)
    kinds = list(rng.choice(["revolute", "continuous", "prismatic"], B - 1))
    if B > 1 and "prismatic" not in kinds:
        kinds[int(rng.integers(0, B - 1))] = "prismatic"
    b.joint_kinds = [""] + kinds
    for i, k in enumerate(kinds, 1):
        if k == "prismatic":
            b.lower[i], b.upper[i], b.limited[i] = -rng.uniform(0.02, 0.15), rng.uniform(0.02, 0.15), True
        elif k == "revolute" and rng.uniform() < 0.5:
            b.lower[i], b.upper[i], b.limited[i] = -0.6, 0.6, True
    b.effort_limit = np.where(rng.uniform(size=B) < 0.5, rng.uniform(0.05, 0.5, B), 0.0)
    b.effort_limit[0] = 0.0
    D = B - 1
    k = rng.uniform(0.0, 5.0, D) if drive else np.zeros(D)
    d = rng.uniform(0.0, 0.05, D) if drive else np.zeros(D)
    modes = ["effort" if (effort and rng.uniform() < 0.35) else "position" for _ in range(D)]
    return ArticulationSpec(b, k, d, rng.integers(0, B, M), np.array([random_rotation(rng) for _ in range(M)]),
                            rng.uniform(-0.1, 0.1, (M, 3)), rng.uniform(-0.02, 0.02, M), drive_mode=modes)


def quad_slider():
    import aerial_gym_simulator_b200.robots  # noqa: F401
    from aerial_gym_simulator_b200.config.env_config import EmptyEnvCfg
    from aerial_gym_simulator_b200.registry._core import robot_registry
    robot, _ = robot_registry.make_robot(ROBOT, "lee_attitude_control", EmptyEnvCfg, "cpu")
    return robot, robot.make_articulation()


# ---- 1. body table and host checks ---------------------------------------------------------------------------------------------
def test_quad_slider_body_table():
    model = urdf.parse_urdf(os.path.join(QUAD, "quad_slider.urdf"))
    assert model.body_order()[5:9] == ["motor_0", "motor_1", "motor_2", "motor_3"]  # application_mask [5, 6, 7, 8] still the motors
    b = model.articulation()
    assert b.num_bodies == 2 and b.joint_kinds == ["", "prismatic"] and b.joint_names[1] == "payload_rail_joint"
    assert b.limited[1] and (b.lower[1], b.upper[1]) == (-0.05, 0.05) and b.effort_limit[1] == 1.0
    np.testing.assert_allclose(b.axis[1], [1, 0, 0])
    np.testing.assert_allclose(b.joint_p[1], [0, 0, -0.03])
    assert b.mass[1] == pytest.approx(0.05) and b.mass[0] == pytest.approx(0.25)
    _, art = quad_slider()
    assert art.prismatic_mask() == 0b10 and list(art.motor_body) == [0, 0, 0, 0]
    assert art.stiffness[0] == 10.0 and art.damping[0] == 0.9


def _slider_urdf(tmp_path, limit, mass=0.05):
    lim = f'<limit lower="{limit[0]}" upper="{limit[1]}" effort="1"/>' if limit else ""
    p = tmp_path / "s.urdf"
    p.write_text(f'<robot name="s"><link name="base"><inertial><mass value="1"/><inertia ixx="1e-3" iyy="1e-3" izz="1e-3" ixy="0" '
                 f'ixz="0" iyz="0"/></inertial></link><link name="p"><inertial><mass value="{mass}"/><inertia ixx="0" iyy="0" izz="0" '
                 f'ixy="0" ixz="0" iyz="0"/></inertial></link><joint name="rail" type="prismatic"><parent link="base"/>'
                 f'<child link="p"/><axis xyz="0 2 0"/>{lim}</joint></robot>')
    return urdf.parse_urdf(str(p))


def test_prismatic_needs_a_bounded_limit(tmp_path):
    for limit in (None, (0.1, 0.1), (0.2, -0.2)):
        with pytest.raises(ValueError, match="^joint 'rail' is prismatic"):
            _slider_urdf(tmp_path, limit).articulation()
    b = _slider_urdf(tmp_path, (-0.1, 0.2)).articulation()
    assert b.joint_kinds[1] == "prismatic" and b.limited[1] and (b.lower[1], b.upper[1]) == (-0.1, 0.2)
    np.testing.assert_allclose(b.axis[1], [0, 1, 0])  # normalised as a revolute axis is


def test_massless_driveless_slider_raises(tmp_path):
    b = _slider_urdf(tmp_path, (-0.1, 0.1), mass=0.0).articulation()
    mk = lambda k, d: ArticulationSpec(b, k, d, [0] * 4, np.tile(np.eye(3), (4, 1, 1)), np.zeros((4, 3)), np.zeros(4))
    with pytest.raises(ValueError, match="joint 'rail': its subtree has no mass to slide"):
        mk(0.0, 0.0)
    mk(1.0, 0.0)
    mk(0.0, 0.1)
    # a massive slider needs no drive, even with no rotational inertia at all
    ArticulationSpec(_slider_urdf(tmp_path, (-0.1, 0.1)).articulation(), 0.0, 0.0, [0] * 4, np.tile(np.eye(3), (4, 1, 1)),
                     np.zeros((4, 3)), np.zeros(4))


# ---- 2. the oracle with sliders --------------------------------------------------------------------------------------------------
def _oracle_table(rng, B, prismatic_share=0.5):
    art = mixed_art(rng, B)
    t = ptable(art.to_struct(), art.prismatic_mask())
    t["prismatic"][1:] |= rng.uniform(size=B - 1) < prismatic_share
    return art, t


def test_oracle_reduces_to_the_revolute_oracles_bit_for_bit():
    """without a slider (no "prismatic" column, or one all False) every function of the prismatic oracle gives its sibling's
    result bit for bit: the dynamics (with effort DOFs), the joint forces, the body motion, the body states and the momentum"""
    rng = np.random.default_rng(3)
    grav, dt = np.array([0.0, 0.0, -9.81]), 0.01
    for _ in range(10):
        B = int(rng.integers(2, 17))
        art, t = _oracle_table(rng, B)
        t.pop("prismatic")
        D = B - 1
        root, q, qd, qs, qds = random_root(rng), rng.uniform(-1, 1, D), rng.uniform(-2, 2, D), rng.uniform(-1, 1, D), rng.uniform(-1, 1, D)
        th, F, T = rng.uniform(0, 2, 4), rng.uniform(-1, 1, 3), rng.uniform(-0.05, 0.05, 3)
        eff = {"effort_dof": rng.uniform(size=D) < 0.5, "effort": rng.uniform(-0.1, 0.1, D), "effort_limit": np.full(D, 0.05)}
        for tab in (t, dict(t, prismatic=np.zeros(B, bool))):
            same = lambda x, y: all(np.array_equal(a, b) for a, b in zip(x, y))
            assert same(PO.dynamics(tab, root, q, qd, qs, qds, dt, grav, th, F, T), AO.dynamics(t, root, q, qd, qs, qds, dt, grav, th, F, T))
            assert same(PO.dynamics(tab, root, q, qd, qs, qds, dt, grav, th, F, T, **eff),
                        EO.dynamics(t, root, q, qd, qs, qds, dt, grav, th, F, T, **eff))
            a, b = PO.joint_force(tab, root, q, qd, qs, qds, dt, grav, th, F, T), JO.joint_force(t, root, q, qd, qs, qds, dt, grav, th, F, T)
            assert all(np.array_equal(a[k], b[k]) for k in a)
            assert same(PO.body_motion(tab, root, q, qd, a["a0"], a["qdd"]), IO.body_motion(t, root, q, qd, a["a0"], a["qdd"]))
            assert np.array_equal(PO.body_states(tab, root, q, qd), BO.body_states(t, root, q, qd))
            assert same(PO.momentum(tab, root, q, qd), AO.momentum(t, root, q, qd))


def _free_model(dt):
    return H.oracle_model_from_spec(MultirotorSpec(controller=_lib.CTRL_NONE, dt=dt, gravity=(0.0, 0.0, 0.0), mass=1.0,
                                                   inertia=np.eye(3), linear_damping=0.0, angular_damping=0.0,
                                                   max_linear_velocity=1e9, max_angular_velocity=1e9))


def test_oracle_free_two_body_slider_period():
    """base 0.25 kg and a 0.05 kg slider whose axis runs through both COMs, a spring k = 10 N / m, no gravity: the two bodies
    oscillate against each other with the period 2 pi sqrt(mu / k) of their reduced mass mu, nothing rotates and the COM stays put"""
    m1, m2, k, dt = 0.25, 0.05, 10.0, 5e-4
    ax = np.array([0.6, 0.0, 0.8])
    t = {"num_bodies": 2, "parent": np.array([-1, 0]), "joint_R": np.array([np.eye(3)] * 2), "joint_p": np.array([[0, 0, 0], ax * 0.05]),
         "axis": np.array([[0, 0, 0], ax]), "mass": np.array([m1, m2]), "com": np.zeros((2, 3)),
         "inertia": np.array([np.eye(3) * 1e-3, np.eye(3) * 1e-5]), "stiffness": np.array([0.0, k]), "damping": np.zeros(2),
         "motor_body": np.zeros(0, int), "motor_R": np.zeros((0, 3, 3)), "motor_p": np.zeros((0, 3)), "motor_torque": np.zeros(0),
         "lower": np.zeros(2), "upper": np.zeros(2), "limited": np.zeros(2, bool), "prismatic": np.array([False, True])}
    model = _free_model(dt)
    root = np.zeros(13)
    root[6] = 1.0
    q, qd = np.array([0.02]), np.zeros(1)
    com = lambda r, q: (m1 * r[0:3] + m2 * (r[0:3] + AO.quat_to_matrix(r[3:7]) @ (t["joint_p"][1] + ax * q[0]))) / (m1 + m2)
    c0 = com(root, q)
    qs, z3 = [], np.zeros(3)
    for _ in range(int(2.0 / dt)):
        a0, qdd = PO.dynamics(t, root, q, qd, np.zeros(1), np.zeros(1), dt, z3, np.zeros(0), z3, z3)
        root, q, qd, _ = AO.integrate(model, t, root, a0, q, qd, qdd)
        qs.append(q[0])
        assert np.abs(root[10:13]).max() < 1e-12 and np.abs(root[3:6]).max() < 1e-12
    assert np.abs(com(root, q) - c0).max() < 1e-9
    qs = np.array(qs)
    up = np.nonzero((qs[:-1] < 0) & (qs[1:] >= 0))[0]
    T = np.diff(up + (-qs[up]) / (qs[up + 1] - qs[up])).mean() * dt
    mu = m1 * m2 / (m1 + m2)
    assert abs(T / (2 * math.pi * math.sqrt(mu / k)) - 1) < 0.01, T


def _energy(t, root, q, qd, qs):
    R, P, S = PO.kinematics(t, root[3:7], q)
    v, e = [None] * int(t["num_bodies"]), 0.0
    for i in range(int(t["num_bodies"])):
        v[i] = np.concatenate([root[10:13], root[7:10]]) if i == 0 else v[int(t["parent"][i])] + S[i] * qd[i - 1]
        I = AO.body_inertia(float(t["mass"][i]), P[i] + R[i] @ t["com"][i], R[i] @ t["inertia"][i] @ R[i].T)
        e += 0.5 * v[i] @ I @ v[i]
    return e + 0.5 * float(np.sum(t["stiffness"][1:len(q) + 1] * (q - qs) ** 2))


def test_oracle_free_trees_with_internal_prismatic_drives_conserve_momentum_and_energy():
    """gravity off, no motors, undamped drives (springs towards fixed targets) on trees mixing the three kinds: the drift of linear
    momentum, of angular momentum about the COM and of the energy (kinetic + spring) over 0.2 s is a first-order integration error:
    halving dt takes at least 40 % off each (0.54 x measured on these trees, the rest second-order terms)"""
    rng = np.random.default_rng(12)
    for B in (3, 6):
        art, t = _oracle_table(rng, B, prismatic_share=0.6)
        t["damping"][:] = 0.0
        t["limited"][:] = False
        t["motor_body"] = np.zeros(0, int)
        D = B - 1
        root0, q0, qd0, qs = random_root(rng), rng.uniform(-0.05, 0.05, D), rng.uniform(-0.5, 0.5, D), rng.uniform(-0.05, 0.05, D)
        root0[7:13] *= 0.2
        drifts = []
        for dt in (0.002, 0.001):
            model = _free_model(dt)
            root, q, qd, z3 = root0.copy(), q0.copy(), qd0.copy(), np.zeros(3)
            p0, L0 = PO.momentum(t, root, q, qd)
            E0 = _energy(t, root, q, qd, qs)
            for _ in range(int(round(0.2 / dt))):
                a0, qdd = PO.dynamics(t, root, q, qd, qs, np.zeros(D), dt, z3, np.zeros(0), z3, z3)
                root, q, qd, _ = AO.integrate(model, t, root, a0, q, qd, qdd)
            p1, L1 = PO.momentum(t, root, q, qd)
            drifts.append((np.linalg.norm(p1 - p0), np.linalg.norm(L1 - L0), abs(_energy(t, root, q, qd, qs) - E0)))
        (pa, la, ea), (pb, lb, eb) = drifts
        assert pb <= 0.6 * pa + 1e-9 and lb <= 0.6 * la + 1e-10 and eb <= 0.6 * ea + 1e-9, drifts


def test_oracle_dof_force_identity_and_base_balance_with_sliders():
    """dof_force of a prismatic DOF (the force along the slide) and of every other DOF = its drive law at the unprojected
    end-of-step state to 1e-12, and the base's Newton-Euler balance to 1e-9, on random trees with sliders, with effort DOFs or not"""
    rng = np.random.default_rng(21)
    grav, dt = np.array([0.0, 0.0, -9.81]), 0.01
    for _ in range(40):
        B = int(rng.integers(2, 17))
        art, t = _oracle_table(rng, B)
        D = B - 1
        root, q, qd, qs, qds = random_root(rng), rng.uniform(-1, 1, D), rng.uniform(-2, 2, D), rng.uniform(-1, 1, D), rng.uniform(-1, 1, D)
        th, F, T = rng.uniform(0, 2, 4), rng.uniform(-1, 1, 3), rng.uniform(-0.05, 0.05, 3)
        eff = rng.uniform(size=D) < 0.5
        t["stiffness"][1:B][eff] = 0.0
        e, lim = rng.uniform(-0.1, 0.1, D), np.where(rng.uniform(size=D) < 0.5, 0.05, 0.0)
        for kw in ({}, {"effort_dof": eff, "effort": e, "effort_limit": lim}):
            o = PO.joint_force(t, root, q, qd, qs, qds, dt, grav, th, F, T, **kw)
            ref = JO.drive_torque(t, q, qd, qs, qds, o["qdd"], dt, **kw)
            assert np.abs(o["dof"] - ref).max() <= 1e-12 * (1 + np.abs(ref).max()), (o["dof"], ref)
            scale = 1 + np.abs(th).sum() + np.abs(F).max() + 9.81 * t["mass"].sum()
            assert np.abs(o["residual"]).max() <= 1e-9 * scale, o["residual"]
            # a prismatic row's torque is about the joint origin, which moves with q: the slide carries no torque of its own
            W = o["wrench"]
            assert all(abs(float(t["axis"][i] @ W[i, :3]) - o["dof"][i - 1]) < 1e-12 * (1 + abs(o["dof"][i - 1]))
                       for i in range(1, B) if t["prismatic"][i])


# ---- 3. the shadow against the oracle on mixed trees ---------------------------------------------------------------------------
def run_prismatic(spec, art, inp, imu_body=None, joint_force=True, effort=None, physics_steps=1):
    n = inp["root"].shape[0]
    eng = CpuPrismaticHp1Engine(spec, n, per_env_params="all", articulation=art, imu_body=imu_body, joint_force=joint_force)
    assert eng._art_step_args()[0] == ("agx_hp1_articulated_step_prismatic" if art.prismatic_mask() else
                                       "agx_hp1_articulated_step_joint_force" if joint_force else "agx_hp1_articulated_step_effort")
    load_inputs(eng, inp)
    if eng.dof_actuation_force is not None:
        eng.dof_actuation_force.copy_(effort)
    eng.physics_step(inp["actions"], disturbance=inp["dist"], physics_steps=physics_steps)
    return eng


def reference(eng, spec, art, inp, idx, effort=None):
    """PO.substep on envs idx with the joint kinds, and the per-env forces: -> (ref dict, ok mask, model, st, table, thrust, F_w, T_w)"""
    model, st = oracle_state(eng, spec, inp, idx)
    ok = H.well_conditioned(model, st, inp["actions"][idx].double()).numpy()
    dof = inp["dof"][idx].double().numpy()
    t = ptable(eng.art, art.prismatic_mask())
    D = art.num_dofs
    e = np.zeros((len(idx), D)) if effort is None else effort[idx].double().numpy()
    lim = np.float32(art.effort_limit).astype(np.float64)
    ref = PO.substep(model, t, st, dof[..., 0], dof[..., 1], inp["qs"][idx].double().numpy(), inp["qds"][idx].double().numpy(),
                     inp["actions"][idx].double(), art.effort_dof, e, lim, inp["dist"][idx].double())
    thrust, F_w, T_w = IO.substep_inputs(model, st, inp["actions"][idx].double(), inp["dist"][idx].double())
    return ref, ok, model, st, t, thrust, F_w, T_w


def slider_tolerances(t, root, q, qd, a0, qdd, grav, thrust, F_w, imu_body):
    """(imu_tolerance, jf_tolerance) of the IMU and joint-force tests, derived from each body's motion, which they read through
    articulated_imu_oracle.body_motion: here that motion is the prismatic oracle's (the same function where nothing slides)"""
    saved = IO.body_motion
    IO.body_motion = PO.body_motion
    try:
        return imu_tolerance(t, imu_body, root, q, qd, a0, qdd, grav), jf_tolerance(t, root, q, qd, a0, qdd, grav, thrust, F_w)
    finally:
        IO.body_motion = saved


def check_all(eng, spec, art, inp, idx, imu_body, effort=None, worst=None):
    """state, IMU input and joint forces of envs idx against the oracle, with the tolerances the other articulated tests derive"""
    ref, ok, model, st, t, thrust, F_w, T_w = reference(eng, spec, art, inp, idx, effort)
    check_substep(eng, spec, inp, ref, ok, idx, worst)
    dof = inp["dof"][idx].double().numpy()
    imu = eng.imu_input.detach().cpu().double().numpy()[idx] if eng.imu_input is not None else None
    W = eng.joint_wrench.detach().cpu().double().numpy()[idx] if eng.joint_wrench is not None else None
    Fd = eng.dof_force.detach().cpu().double().numpy()[idx] if eng.joint_wrench is not None else None
    for k in np.flatnonzero(ok):
        r, q, qd, a0, qdd = st.root[k].numpy(), dof[k, :, 0], dof[k, :, 1], ref["a0"][k], ref["qdd"][k]
        imu_tol, jf_tol = slider_tolerances(t, r, q, qd, a0, qdd, model.gravity, thrust[k], F_w[k], imu_body)
        motion = PO.body_motion(t, r, q, qd, a0, qdd)
        if imu is not None:
            err, tol = np.abs(imu[k] - IO.imu_from_motion(t, imu_body, model.gravity, *motion)), \
                imu_tol
            assert (err <= tol).all(), ("imu", k, err, tol)
        if W is not None:
            f, R, P = PO.newton_euler(t, r, q, qd, a0, qdd, model.gravity, thrust[k], F_w[k], T_w[k])
            wr, dr = PO.rows(t, f, R, P)
            tol = jf_tol
            assert (np.abs(W[k] - wr) <= tol).all(), ("joint_wrench", k, np.abs(W[k] - wr), tol)
            # a prismatic DOF's force is the force component of its row: the row's force tolerance
            tdof = np.where(t["prismatic"][1:], tol[1:, 0], tol[1:, 3])
            assert (np.abs(Fd[k] - dr) <= tdof).all(), ("dof_force", k, np.abs(Fd[k] - dr), tdof)
    if W is not None:
        assert (W[:, 0] == 0).all()
        check_dof_force_identity(eng, art, inp, np.asarray(idx)[ok], effort)
    return ok


@pytest.mark.parametrize("M", [4, 8])
def test_shadow_matches_oracle_on_mixed_trees(M):
    """random trees of 1-16 bodies mixing the three joint kinds, drives on and off, effort DOFs, the IMU on the base, a middle body
    and a leaf, joint forces on and off, and joints started inside and at both limits with velocities pointing out"""
    rng = np.random.default_rng(60 + M)
    spec = H.spec_for("quad_attitude" if M == 4 else "octa_velocity")
    worst = {}
    for trial in range(16):
        B = trial + 1
        art = mixed_art(rng, B, M=M, drive=bool(trial % 2), effort=trial % 3 == 0)
        n = 24
        for variant in range(2):
            inp = substep_inputs(spec, art, n, 300 + 2 * trial + variant)
            if variant:
                inp = _limit_crossing(inp, art)
            eff = torch.tensor(rng.uniform(-0.6, 0.6, (n, B - 1)), dtype=torch.float32)
            imu_body = [0, B // 2, B - 1][(trial + variant) % 3]
            eng = run_prismatic(spec, art, inp, imu_body=imu_body, joint_force=bool((trial + variant) % 2 == 0) or B == 1, effort=eff)
            ok = check_all(eng, spec, art, inp, np.arange(n), imu_body, eff if art.effort_dof.any() else None, worst)
            assert ok.mean() > 0.8
            if variant and art.bodies.limited.any():
                q = eng.dof_state[..., 0].double().numpy()
                lim = art.bodies.limited[1:]
                assert ((q[:, lim] == np.float32(art.bodies.upper[1:][lim])) | (q[:, lim] == np.float32(art.bodies.lower[1:][lim]))).any()
    print({k: f"{v[0]:.2f} ({v[1]:.1e})" for k, v in worst.items()})


def test_physics_steps_zero():
    """no sub-step: state unchanged, joint forces and the IMU's force inputs zero, its w_b the unstepped state's (through a slider)"""
    spec = H.spec_for("quad_attitude")
    rng = np.random.default_rng(4)
    art = mixed_art(rng, 6)
    inp = substep_inputs(spec, art, 16, 9)
    b = 5
    eng = run_prismatic(spec, art, inp, imu_body=b, physics_steps=0)
    assert torch.equal(eng.root_state, inp["root"]) and torch.equal(eng.dof_state, inp["dof"])
    assert (eng.joint_wrench == 0).all() and (eng.dof_force == 0).all() and (eng.imu_input[:, :6] == 0).all()
    t = ptable(eng.art, art.prismatic_mask())
    for k in range(16):
        r, dof = inp["root"][k].double().numpy(), inp["dof"][k].double().numpy()
        R, P, V, _ = PO.body_motion(t, r, dof[:, 0], dof[:, 1], np.zeros(6), np.zeros(5))
        np.testing.assert_allclose(eng.imu_input[k, 6:].double().numpy(), R[b].T @ V[b, :3], atol=1e-5 * (1 + np.abs(V[b, :3]).max()))


# ---- 4. revolute-only trees: the prismatic entry is the other steps, bit for bit (no FMA contraction on the host) --------------
@pytest.mark.parametrize("B", [1, 2, 9, 10, 16])
def test_revolute_tree_through_prismatic_entry_is_bit_identical(B):
    rng = np.random.default_rng(80 + B)
    spec = H.spec_for("quad_attitude")
    art = mixed_art(rng, B)
    art.bodies.joint_kinds = [""] + ["revolute"] * (B - 1)
    art.bodies.limited[1:] = False
    art = with_effort(art, rng)
    n = 32
    inp = substep_inputs(spec, art, n, 7 + B)
    eff = torch.tensor(rng.uniform(-0.3, 0.3, (n, B - 1)), dtype=torch.float32)
    lib = _articulated_prismatic_shadow.load()
    for imu_body, jf in ((None, False), (B - 1, False), (None, True), (B // 2, True)):
        ref = CpuPrismaticHp1Engine(spec, n, per_env_params="all", articulation=art, imu_body=imu_body, joint_force=jf)
        got = CpuPrismaticHp1Engine(spec, n, per_env_params="all", articulation=art, imu_body=imu_body, joint_force=jf)
        for e in (ref, got):
            load_inputs(e, inp)
            if e.dof_actuation_force is not None:
                e.dof_actuation_force.copy_(eff)
        ref.physics_step(inp["actions"], disturbance=inp["dist"], physics_steps=3)
        got._set_inputs(inp["actions"].contiguous(), inp["dist"], 3, None, 0)
        effort = got._effort_ref if got._effort is not None else None
        imu = (imu_body, got.imu_input.data_ptr()) if imu_body is not None else (0, None)
        out = (got.joint_wrench.data_ptr(), got.dof_force.data_ptr()) if jf else (None, None)
        assert lib.shadow_art_step_prismatic(got._cfg_ref, got._buf_ref, got._art_ref, 0, effort, *imu, *out) == 0
        for k in ("root_state", "motor_thrust", "dof_state", "imu_input", "joint_wrench", "dof_force") + CpuPrismaticHp1Engine.DERIVED:
            a, b = getattr(ref, k), getattr(got, k)
            assert (a is None) == (b is None), k
            if a is not None:
                assert torch.equal(a, b), (k, imu_body, jf)
        # the body states through the prismatic entry, too
        ref.update_body_state()
        bs = torch.zeros_like(got.body_state)
        _articulated_prismatic_shadow.load().shadow_art_body_state_prismatic(C.byref(got.art), 0, n, got.root_state.data_ptr(), 13, bs.data_ptr())
        assert torch.equal(ref.body_state, bs)


def with_effort(art, rng):
    modes = ["effort" if rng.uniform() < 0.4 else "position" for _ in range(art.num_dofs)]
    return dataclasses.replace(art, drive_mode=modes, effort_limit=None)


# ---- 5. body states ------------------------------------------------------------------------------------------------------------
def test_body_states_match_oracle_on_mixed_trees():
    """every row against articulated_body_state_oracle with the kinds: a prismatic row keeps its parent's joint-frame rotation, its
    origin moves by a q and its velocity by a q-dot.  Bar: 32 eps per level of depth on the row's magnitudes (the rotation's
    rounding, as in the body-state tests), plus the world position's ulps"""
    rng = np.random.default_rng(5)
    n = 16
    for B in (1, 2, 5, 9, 10, 16):
        art = mixed_art(rng, B)
        s = art.to_struct()
        mask = art.prismatic_mask()
        t = ptable(s, mask)
        root = torch.tensor(np.array([random_root(rng) for _ in range(n)]), dtype=torch.float32)
        dof = torch.tensor(np.stack([rng.uniform(-0.1, 0.1, (n, B - 1)), rng.uniform(-2, 2, (n, B - 1))], -1), dtype=torch.float32)
        s.dof_state = dof.data_ptr()
        out = torch.zeros(n, B, 13)
        _articulated_prismatic_shadow.body_state(s, root, out, mask)
        assert torch.equal(out[:, 0], root)
        for k in range(n):
            ref = PO.body_states(t, root[k].double().numpy(), dof[k, :, 0].double().numpy(), dof[k, :, 1].double().numpy())
            got = out[k].double().numpy()
            for i in range(1, B):
                qs = ref[i, 3:7] if ref[i, 3:7] @ got[i, 3:7] >= 0 else -ref[i, 3:7]
                e = 32 * EPS * (_depth(t, i) + 1)
                pos = np.abs(got[i, 0:3] - ref[i, 0:3]).max()
                assert pos <= e * (np.abs(ref[i, 0:3] - root[k, 0:3].double().numpy()).max() + 1.0) + 4 * EPS * np.abs(ref[i, 0:3]).max(), (B, i, pos)
                assert np.abs(got[i, 3:7] - qs).max() <= e, (B, i)
                vs = np.abs(ref[i, 7:13]).max() + np.abs(ref[:, 10:13]).max() * 1.0 + 1.0
                assert np.abs(got[i, 7:13] - ref[i, 7:13]).max() <= e * vs, (B, i, np.abs(got[i, 7:13] - ref[i, 7:13]).max())


# ---- 6. the stiff limit of the shipped robot -----------------------------------------------------------------------------------
def _fixed_pair(tmp_path, rail_z):
    """(rigid spec, articulation with k = 1e4 N / m) of quad_slider.urdf with its rail at height rail_z: the articulated robot, and
    the same URDF with the rail joint made fixed as a rigid robot"""
    from aerial_gym_simulator_b200.config import robot_config as rc
    from aerial_gym_simulator_b200.config.env_config import EmptyEnvCfg
    from aerial_gym_simulator_b200.registry._core import robot_registry
    from aerial_gym_simulator_b200.robots import ArticulatedMultirotor, BaseMultirotor
    text = open(os.path.join(QUAD, "quad_slider.urdf")).read().replace('<origin xyz="0.0 0.0 -0.03" rpy="0.0 0.0 0.0"/>\n    <axis',
                                                                         f'<origin xyz="0.0 0.0 {rail_z}" rpy="0.0 0.0 0.0"/>\n    <axis')
    out = []
    for kind, cls in (("fixed", BaseMultirotor), ("prismatic", ArticulatedMultirotor)):
        name = f"_test_quad_slider_{kind}_{rail_z}"
        (tmp_path / f"{name}.urdf").write_text(text.replace('type="prismatic"', f'type="{kind}"'))

        class Cfg(rc.BaseQuadWithSlidingPayloadCfg):
            class robot_asset(rc.BaseQuadWithSlidingPayloadCfg.robot_asset):
                asset_folder, file = str(tmp_path), f"{name}.urdf"

        Cfg.robot_asset.name = name
        robot_registry.register(name, cls, Cfg)
        out.append(name)
    spec = spec_from_registry(out[0], "lee_attitude_control")
    art = robot_registry.make_robot(out[1], "lee_attitude_control", EmptyEnvCfg, "cpu")[0].make_articulation()
    art.stiffness[:] = 1e4
    return spec, art


@pytest.mark.parametrize("rail_z", [-0.03, 0.0])
def test_stiff_slider_tracks_the_fixed_payload(tmp_path, rail_z):
    """k = 1e4 N / m and q* = 0 on payload_rail_joint: the payload moves by micrometres, so quad_slider.urdf follows the same URDF
    with the rail joint made fixed, stepped by the rigid HP1 path, over 1 s of random attitude commands: the attitude within 1e-3.
    The rigid step integrates the base origin as the centre of mass (DESIGN.md section 3), which the shipped rail, 3 cm below the
    base origin, moves 5 mm away from it: there the base positions part by that model's own error (4e-3 m on this run), not the
    slider's.  With the rail through the base origin the rigid model is exact, and positions agree within 1e-3 too (5e-6 m)."""
    spec, art = _fixed_pair(tmp_path, rail_z)
    n = 32
    hp1 = CpuHp1Engine(spec, n, per_env_params="all")
    arte = CpuPrismaticHp1Engine(spec, n, per_env_params="all", articulation=art)
    rng = np.random.default_rng(5)
    _random_start((hp1, arte), n, rng, v=0.2, w=0.2)
    for _ in range(10):
        act = torch.from_numpy(rng.uniform(-0.3, 0.3, (n, 4))).float()
        hp1.physics_step(act, physics_steps=10)
        arte.physics_step(act, physics_steps=10)
    assert torch.isfinite(arte.root_state).all()
    assert (arte.root_state[:, 3:7] - hp1.root_state[:, 3:7]).abs().max().item() < 1e-3
    assert arte.dof_state[..., 0].abs().max().item() < 1e-4
    if rail_z == 0.0:
        assert (arte.root_state[:, 0:3] - hp1.root_state[:, 0:3]).abs().max().item() < 1e-3


# ---- 7. host layer on the CPU stack --------------------------------------------------------------------------------------------
def test_sliding_payload_runs_position_task_and_publishes_its_slider(monkeypatch):
    from aerial_gym_simulator_b200.registry._core import task_registry
    import aerial_gym_simulator_b200.task  # noqa: F401
    cfg = task_registry.get_task_config("position_setpoint_task")
    monkeypatch.setattr(cfg, "robot_name", ROBOT)
    monkeypatch.setattr(cfg, "device", "cpu")
    with prismatic_cpu_stack():
        task = task_registry.make_task("position_setpoint_task", seed=1, num_envs=16, headless=True)
        assert task._unfused
        task.reset()
        gtd = task.sim_env.global_tensor_dict
        assert gtd["dof_state_tensor"].shape == (16, 1, 2) and gtd["robot_body_state_tensor"].shape == (16, 2, 13)
        gtd["dof_position_setpoint_tensor"].fill_(0.04)
        g = torch.Generator().manual_seed(0)
        for _ in range(40):
            obs, rew, term, trunc, _ = task.step(torch.rand(16, 4, generator=g) * 0.2 - 0.1)
        assert torch.isfinite(obs["observations"]).all() and torch.isfinite(rew).all()
        q = gtd["dof_state_tensor"][:, 0, 0]
        assert (q.abs() <= 0.05).all() and (q > 0.02).all(), q  # the drive has moved the payload towards 4 cm
        # the payload's row: the base's pose moved along its x axis by q, 3 cm below the base origin
        rows, root = gtd["robot_body_state_tensor"], gtd["robot_state_tensor"]
        R = torch.stack([torch.tensor(AO.quat_to_matrix(r[3:7].double().numpy())) for r in root])
        p = root[:, 0:3].double() + (R @ torch.stack([q.double(), torch.zeros(16, dtype=torch.float64), torch.full((16,), -0.03,
                                                                                                               dtype=torch.float64)], 1)[..., None])[..., 0]
        assert (rows[:, 1, 0:3].double() - p).abs().max().item() < 1e-5
        assert (rows[:, 1, 3:7].abs() - root[:, 3:7].abs()).abs().max().item() < 1e-5


# ---- 8. C ABI and machine code -------------------------------------------------------------------------------------------------
def test_c_abi_validation():
    lib = _lib.load()
    spec = H.spec_for("quad_attitude")
    _, art = quad_slider()
    buf, s = _lib.AgxHp1Buffers(), art.to_struct()
    jw, df = torch.zeros(64, 2, 6), torch.zeros(64, 4)
    call = lambda n, mask=2, w=None, d=None, st=s, b=0, im=None: lib.agx_hp1_articulated_step_prismatic(
        C.byref(build_config(spec, n)), C.byref(buf), C.byref(st), mask, None, b, im, w, d, None)
    bst = lambda mask, st=s, out=jw.data_ptr(), n=0: lib.agx_hp1_articulated_body_state_prismatic(C.byref(st), mask, n, jw.data_ptr(),
                                                                                                  13, out, None)
    assert call(0) == 0 and call(0, w=jw.data_ptr(), d=df.data_ptr()) == 0
    for mask, what in ((3, b"bit 0"), (6, b"at or above num_bodies")):
        assert call(0, mask) != 0 and what in lib.agx_last_error()
        assert bst(mask) != 0 and what in lib.agx_last_error()
    for lo, hi, limited in ((0.1, 0.1, 1), (-0.05, 0.05, 0)):
        s2 = art.to_struct()
        s2.lower[1], s2.upper[1], s2.limited[1] = lo, hi, limited
        assert call(0, st=s2) != 0 and b"body 1's joint is prismatic" in lib.agx_last_error()
        assert bst(2, st=s2) != 0 and b"body 1's joint is prismatic" in lib.agx_last_error()
    assert call(0, b=2, im=jw.data_ptr()) != 0 and b"imu_body" in lib.agx_last_error()
    x = torch.zeros(64)
    buf.root_state, buf.motor_thrust, buf.actions = x.data_ptr(), x.data_ptr(), x.data_ptr()
    s.dof_state = s.dof_position_setpoint = s.dof_velocity_setpoint = x.data_ptr()
    assert call(1, d=df.data_ptr()) != 0 and b"without joint_wrench" in lib.agx_last_error()
    assert call(1, w=jw.data_ptr()) != 0 and b"dof_force is NULL" in lib.agx_last_error()
    for w, d in ((jw.data_ptr() + 8, df.data_ptr()), (jw.data_ptr(), df.data_ptr() + 4)):
        assert call(1, w=w, d=d) != 0 and b"16-byte aligned" in lib.agx_last_error()
    assert bst(2, out=jw.data_ptr() + 4, n=1) != 0 and b"16-byte aligned" in lib.agx_last_error()


def test_prismatic_kernels_have_no_spills():
    """articulated_prismatic.cu's six kernels under -Xptxas -v: no spills; the body-state kernels use no stack either"""
    src = os.path.join(_build.CSRC, "articulated_prismatic.cu")
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.run([_build._nvcc()] + _build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o", os.path.join(d, "p.o")],
                           capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    blocks = re.findall(r"Compiling entry function '(\S+)'.*?\n.*?(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads",
                        r.stderr, re.S)
    names = sorted(re.search(r"\d(articulated_(?:step|body_state)_prismatic_kernelILi\d+E(?:Li\d+E)?)", f).group(1) for f, *_ in blocks)
    assert names == sorted([f"articulated_step_prismatic_kernelILi{m}ELi{nb}E" for m in (4, 8) for nb in (9, 16)] +
                           [f"articulated_body_state_prismatic_kernelILi{nb}E" for nb in (9, 16)]), names
    for f, stack, st, ld in blocks:
        assert st == "0" and ld == "0", f
        if "body_state" in f:
            assert stack == "0", f
