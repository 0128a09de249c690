"""Joint force sensing of articulated robots on the CPU (DESIGN.md "Articulated robots", "Joint force sensing"): joint_wrench and
dof_force of art_env_step<M, NB, true, true, true> (host shadow, tests/csrc/articulated_joint_force_shadow.cu) against
oracle/articulated_joint_force_oracle.py, the oracle's own checks (the dof_force identity, the base's Newton-Euler balance, a hanging
pendulum, a one-body tree), bit identity of the state with the plain, IMU and effort steps, static loads at hover, and the host layer
(Hp1Engine, EnvManager, the C ABI) on the CPU stack."""
import ctypes as C
import dataclasses
import re

import numpy as np
import pytest
import torch

from aerial_gym_simulator_b200 import _lib
from aerial_gym_simulator_b200.hp1 import build_config
from oracle import articulated_imu_oracle as IO
from oracle import articulated_joint_force_oracle as JO
from oracle import hp1_oracle as HO

from . import _hp1_common as H
from ._cpu_stack_articulated import CpuArticulatedHp1Engine
from ._cpu_stack_articulated_effort import CpuEffortHp1Engine
from ._cpu_stack_articulated_imu import CpuImuHp1Engine
from ._cpu_stack_articulated_joint_force import CpuJointForceHp1Engine, joint_force_cpu_stack
from .test_articulated_cpu import RTOL, load_inputs, morphy_compliant, oracle_state, random_art, random_root, shaped_art, substep_inputs, \
    table_of
from .test_articulated_effort_cpu import articulated_unit, effort_inputs, with_modes  # noqa: F401 (articulated_unit is a fixture)
from .test_articulated_imu_cpu import _depth, _limit_crossing, gimbal_quad, sass_functions

EPS = float(np.finfo(np.float32).eps)
ULPS = 8
STATE = ("root_state", "motor_thrust", "dof_state") + CpuArticulatedHp1Engine.DERIVED


def run_jf(spec, art, inp, physics_steps=1, imu_body=None, effort=None):
    n = inp["root"].shape[0]
    eng = CpuJointForceHp1Engine(spec, n, per_env_params="all", articulation=art, imu_body=imu_body, joint_force=True)
    load_inputs(eng, inp)
    if eng.dof_actuation_force is not None:
        eng.dof_actuation_force.copy_(effort)
    eng.physics_step(inp["actions"], disturbance=inp["dist"], physics_steps=physics_steps)
    return eng


# ---- tolerance -----------------------------------------------------------------------------------------------------------------
# Row i is the sum over the bodies k of body i's subtree of I_k A_k + V_k x* I_k V_k - f_ext,k (the oracle's recursion; the ABA's
# I^A_i A_i + p^A_i is the same sum, gathered by the backward pass).  The float32 ABA gives a0 and every qdd within RTOL amax of the
# float64 solve (test_articulated_cpu.py section 2), so body k's spatial acceleration, d_k + 1 such terms deep, is off by
# E_ang,k = RTOL amax (d_k + 1) in its angular part and E_lin,k = E_ang,k (1 + L) in its linear part, L the largest lever |P| + |c|
# of the tree (test_articulated_imu_cpu.imu_tolerance).  Through I_k: m_k (E_lin,k + E_ang,k L) in the force, and
# (|Ic_k| + m_k L^2) E_ang,k + m_k L E_lin,k in the torque about O.  Every rotation is off by e_R = 32 eps (depth + 1) and each sum
# or product adds ULPS ulps of its terms' magnitude: S_F = sum_k m_k (|a_k| + |alpha_k| L + |w_k| (|v_k| + |w_k| L) + |g|) + the
# thrusts on k (and the drag on the base), S_n = S_F L + sum_k |Ic_k| (|alpha_k| + |w_k|^2) + the motors' reaction torques.  Moving
# the torque from O to the joint origin P_i adds |P_i| times the force's error.
def jf_tolerance(table, root, q, qd, a0, qdd, grav, thrust, F_w):
    B = int(table["num_bodies"])
    R, P, V, A = IO.body_motion(table, root, q, qd, a0, qdd)
    L = max(float(np.linalg.norm(P[i] + R[i] @ table["com"][i])) for i in range(B))
    amax = float(np.abs(np.concatenate([a0, qdd])).max())
    g = float(np.linalg.norm(grav))
    rot = 32 * EPS * (max(_depth(table, i) for i in range(B)) + 1) + ULPS * EPS
    eF, en, sF, sn = np.zeros(B), np.zeros(B), np.zeros(B), np.zeros(B)
    for k in range(B):
        m, Ic = float(table["mass"][k]), float(np.abs(table["inertia"][k]).sum())
        ea = RTOL * amax * (_depth(table, k) + 1)
        el = ea * (1.0 + L)
        w, al = np.linalg.norm(V[k, :3]), np.linalg.norm(A[k, :3])
        eF[k] = m * (el + ea * L)
        en[k] = (Ic + m * L * L) * ea + m * L * el
        sF[k] = m * (np.linalg.norm(A[k, 3:]) + al * L + w * (np.linalg.norm(V[k, 3:]) + w * L) + g)
        sn[k] = Ic * (al + w * w)
    for j, b in enumerate(table["motor_body"][:len(thrust)]):
        sF[int(b)] += abs(float(thrust[j]))
        sn[int(b)] += abs(float(thrust[j] * table["motor_torque"][j]))
    sF[0] += float(np.linalg.norm(F_w))
    tol = np.zeros((B, 6))
    for i in range(B - 1, 0, -1):
        sub = [k for k in range(i, B) if k == i or _ancestor(table, i, k)]
        tF = eF[sub].sum() + rot * sF[sub].sum()
        tn = en[sub].sum() + rot * (sF[sub].sum() * L + sn[sub].sum())
        p = float(np.linalg.norm(P[i]))
        tol[i, :3], tol[i, 3:] = tF, tn + p * tF + rot * p * sF[sub].sum()
    return tol


def _ancestor(table, i, k):
    while k > 0:
        k = int(table["parent"][k])
        if k == i:
            return True
    return False


def check_joint_force(eng, spec, inp, art, idx, effort=None, worst=None):
    """the engine's joint_wrench / dof_force of envs idx against JO.substep at the inputs' state, with jf_tolerance; envs that fail
    _hp1_common.well_conditioned are only checked for finite values.  -> worst err / tol"""
    model, st = oracle_state(eng, spec, inp, idx)
    ok = H.well_conditioned(model, st, inp["actions"][idx].double()).numpy()
    dof = inp["dof"][idx].double().numpy()
    table = table_of(eng.art)
    e = None if effort is None else effort[idx].double().numpy()
    kw = {} if effort is None else {"effort_dof": art.effort_dof, "effort": e,
                                    "effort_limit": np.float32(art.effort_limit).astype(np.float64)}
    ref = JO.substep(model, table, st, dof[..., 0], dof[..., 1], inp["qs"][idx].double().numpy(), inp["qds"][idx].double().numpy(),
                     inp["actions"][idx].double(), inp["dist"][idx].double(), **kw)
    W = eng.joint_wrench.detach().cpu().double().numpy()[idx]
    Fd = eng.dof_force.detach().cpu().double().numpy()[idx]
    assert np.isfinite(W).all() and np.isfinite(Fd).all()
    assert (W[:, 0] == 0).all()
    thrust, F_w, _ = IO.substep_inputs(model, st, inp["actions"][idx].double(), inp["dist"][idx].double())
    r = 0.0
    for k in np.flatnonzero(ok):
        tol = jf_tolerance(table, st.root[k].numpy(), dof[k, :, 0], dof[k, :, 1], ref["a0"][k], ref["qdd"][k], model.gravity, thrust[k],
                           F_w[k])
        err = np.abs(W[k] - ref["wrench"][k])
        assert (err <= tol).all(), (k, err, tol)
        et = np.abs(Fd[k] - ref["dof"][k])
        assert (et <= tol[1:, 3]).all(), (k, et, tol[1:, 3])
        r = max(r, float(np.max(err[1:] / tol[1:], initial=0.0)), float(np.max(et / tol[1:, 3], initial=0.0)))
    if worst is not None:
        worst.append(r)
    check_dof_force_identity(eng, art, inp, idx[ok] if len(idx) else idx, effort)
    return r


# The dof_force identity on the step's own outputs (one sub-step): DOF j's force is the drive law at the end-of-step state the step
# wrote, k (q* - q') + d (q-dot* - q-dot') for a position DOF and tau_e - d q-dot' for an effort DOF, with q', q-dot' read back from
# dof_state -- except where the step projected the joint onto a limit, which replaces q', q-dot'.  Independent of the oracle, and
# tight: both sides are float32 sums of the same terms, so the bar is IDENTITY_ULPS float32 ulps of the largest of them -- the drive's
# terms, its implicit part (d + dt k) |q-dot' - q-dot|, and the torques the ABA sums for the joint about O, which are bounded by the
# joint's wrench row (|n_i| + |P_i| |F_i|) and the explicit drive.
IDENTITY_ULPS = 256


def check_dof_force_identity(eng, art, inp, idx, effort=None):
    if art.num_dofs == 0 or len(idx) == 0:
        return 0.0
    table, dt = table_of(eng.art), float(eng.cfg.dt)
    B = art.num_dofs + 1
    k, d = table["stiffness"][1:B], table["damping"][1:B]
    out = eng.dof_state.detach().cpu().double().numpy()[idx]
    q1, v1 = out[..., 0], out[..., 1]
    q0, v0 = inp["dof"][idx].double().numpy()[..., 0], inp["dof"][idx].double().numpy()[..., 1]
    qs, qds = inp["qs"][idx].double().numpy(), inp["qds"][idx].double().numpy()
    got = eng.dof_force.detach().cpu().double().numpy()[idx]
    W = eng.joint_wrench.detach().cpu().double().numpy()[idx][:, 1:]
    # the torque about O that the row's torque comes from: |n_i| + |P_i| |F_i|, |P_i| at most the joint offsets along the path
    lever = np.zeros(B)
    for i in range(1, B):
        lever[i] = lever[int(table["parent"][i])] + float(np.linalg.norm(table["joint_p"][i]))
    n = np.abs(W[..., 3:]).max(-1) + lever[1:] * np.linalg.norm(W[..., :3], axis=-1)
    pos = k * (qs - q1) + d * (qds - v1)
    scale = np.abs(k * qs) + np.abs(k * q1) + np.abs(d * qds) + np.abs(d * v1) + (d + dt * k) * np.abs(v1 - v0) + \
        k * (np.abs(q0) + dt * np.abs(v0)) + n
    if effort is not None and art.effort_dof.any():
        te = JO.EO.effort_torque(effort[idx].double().numpy(), np.float32(art.effort_limit).astype(np.float64))
        ref = np.where(art.effort_dof, te - d * v1, pos)
        scale = scale + np.abs(te)
    else:
        ref = pos
    lim = table["limited"][1:B].astype(bool)
    projected = lim & ((q1 == np.float32(table["lower"][1:B])) | (q1 == np.float32(table["upper"][1:B])))
    err = np.where(projected, 0.0, np.abs(got - ref))
    tol = IDENTITY_ULPS * EPS * scale
    assert (err <= tol).all(), (np.argwhere(err > tol)[:4], (err / tol).max())
    return float((err / tol).max())


# ---- the oracle itself ---------------------------------------------------------------------------------------------------------
def _case(rng, B, M=4):
    art = random_art(rng, B, M=M)
    D = B - 1
    return art, table_of(art.to_struct()), random_root(rng), rng.uniform(-1, 1, D), rng.uniform(-2, 2, D), rng.uniform(-1, 1, D), \
        rng.uniform(-1, 1, D), rng.uniform(0, 2, M), rng.uniform(-1, 1, 3), rng.uniform(-0.05, 0.05, 3)


def test_oracle_dof_force_identity_and_base_balance():
    """dof_force = k (q* - q') + d (q-dot* - q-dot') (position) or tau_e - d q-dot' (effort) to 1e-12, and the base's Newton-Euler
    balance (thrusts, drag and gravity on body 0 minus its children's reactions = its rate of momentum) to 1e-9, on random trees"""
    rng = np.random.default_rng(1)
    grav, dt = np.array([0.0, 0.0, -9.81]), 0.01
    for _ in range(40):
        B = int(rng.integers(1, 17))
        art, tab, root, q, qd, qs, qds, th, F, T = _case(rng, B)
        D = B - 1
        eff = rng.uniform(size=D) < 0.5
        tab["stiffness"][1:B][eff] = 0.0
        e, lim = rng.uniform(-0.1, 0.1, D), np.where(rng.uniform(size=D) < 0.5, 0.05, 0.0)
        for kw in ({}, {"effort_dof": eff, "effort": e, "effort_limit": lim}):
            o = JO.joint_force(tab, root, q, qd, qs, qds, dt, grav, th, F, T, **kw)
            ref = JO.drive_torque(tab, q, qd, qs, qds, o["qdd"], dt, **kw)
            assert np.abs(o["dof"] - ref).max(initial=0.0) <= 1e-12 * (1 + np.abs(ref).max(initial=0.0)), (o["dof"], ref)
            scale = 1 + np.abs(th).sum() + np.abs(F).max() + 9.81 * tab["mass"].sum()
            assert np.abs(o["residual"]).max() <= 1e-9 * scale, o["residual"]
            assert (o["wrench"][0] == 0).all()


def test_oracle_hanging_pendulum_carries_its_weight():
    """a base at rest with a rod of mass m on a y-axis joint, its COM l below the pivot, at rest at angle theta.  Held (qdd = 0):
    the joint carries the rod's weight, (0, 0, m g) in world axes, and the moment m g l sin theta about its axis.  Swinging freely
    (qdd = -m g l sin theta / (J + m l^2)): no moment about the axis."""
    m, l, J, g = 0.3, 0.2, 1e-3, 9.81
    z2 = np.zeros(2)
    tab = {"num_bodies": 2, "parent": np.array([-1, 0]), "joint_R": np.array([np.eye(3)] * 2), "joint_p": np.zeros((2, 3)),
           "axis": np.array([[0, 0, 0], [0, 1.0, 0]]), "mass": np.array([1.0, m]), "com": np.array([[0, 0, 0], [0, 0, -l]]),
           "inertia": np.array([np.eye(3) * 1e-3, np.diag([J, J, J])]), "stiffness": z2, "damping": z2, "motor_body": np.zeros(4, int),
           "motor_R": np.array([np.eye(3)] * 4), "motor_p": np.zeros((4, 3)), "motor_torque": np.zeros(4)}
    root = np.zeros(13)
    root[6] = 1.0
    grav, z3 = np.array([0.0, 0.0, -g]), np.zeros(3)
    for th in (0.0, 0.4, -1.0):
        f, R, P = JO.newton_euler(tab, root, [th], [0.0], np.zeros(6), [0.0], grav, np.zeros(4), z3, z3)
        W, dof = JO.rows(tab, f, R, P)
        np.testing.assert_allclose(W[1, :3], R[1].T @ np.array([0, 0, m * g]), atol=1e-12)
        np.testing.assert_allclose(dof, [m * g * l * np.sin(th)], atol=1e-12)
        np.testing.assert_allclose(np.linalg.norm(W[1, :3]), m * g, rtol=1e-12)
        qdd = -m * g * l * np.sin(th) / (J + m * l * l)
        f, R, P = JO.newton_euler(tab, root, [th], [0.0], np.zeros(6), [qdd], grav, np.zeros(4), z3, z3)
        assert abs(JO.rows(tab, f, R, P)[1][0]) < 1e-12  # swinging freely, nothing acts about the axis


def test_oracle_one_body_tree_has_only_a_zero_row():
    rng = np.random.default_rng(3)
    _, tab, root, q, qd, qs, qds, th, F, T = _case(rng, 1)
    o = JO.joint_force(tab, root, q, qd, qs, qds, 0.01, np.array([0, 0, -9.81]), th, F, T)
    assert o["wrench"].shape == (1, 6) and (o["wrench"] == 0).all() and o["dof"].shape == (0,)
    assert np.abs(o["residual"]).max() <= 1e-9 * (1 + np.abs(th).sum() + np.abs(F).max() + 9.81 * tab["mass"].sum())


# ---- the shadow against the oracle -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("robot", ["morphy_compliant", "gimbal", "torque_gimbal"])
def test_shadow_matches_oracle_on_shipped_robots(robot):
    """drives on (the robot's own gains) and off; joints inside and crossing their limits; the torque gimbal with commands inside
    and beyond its limits"""
    spec = H.spec_for("quad_attitude")
    _, art = morphy_compliant() if robot == "morphy_compliant" else gimbal_quad()
    if robot == "torque_gimbal":
        art = with_modes(art, "effort")
    worst = []
    for drive in (True, False):
        a = art
        if not drive and robot != "torque_gimbal":
            a = dataclasses.replace(art, stiffness=0.0, damping=1e-4)  # morphy's massless connecting links need some drive
        for cross in (False, True):
            inp = substep_inputs(spec, a, 24, 700 + 10 * cross + 20 * drive)
            if cross:
                inp = _limit_crossing(inp, a)
            effort = effort_inputs(a, 24, 701 + cross) if robot == "torque_gimbal" else None
            eng = run_jf(spec, a, inp, effort=effort)
            check_joint_force(eng, spec, inp, a, np.arange(24), effort, worst)
    print(f"worst err/tol {max(worst):.3f}")


@pytest.mark.parametrize("M", [4, 8])
def test_shadow_matches_oracle_on_random_trees(M):
    rng = np.random.default_rng(90 + M)
    spec = H.spec_for("quad_attitude" if M == 4 else "octa_velocity")
    worst = []
    for B in range(1, 17):
        art = shaped_art(rng, B, M=M, drive=bool(B % 2))
        if not B % 2:
            art = dataclasses.replace(art, damping=1e-3)
        art.bodies.limited[1:] = True
        inp = substep_inputs(spec, art, 16, 900 + B)
        if B % 3 == 0:
            inp = _limit_crossing(inp, art)
        eng = run_jf(spec, art, inp)
        check_joint_force(eng, spec, inp, art, np.arange(16), worst=worst)
    print(f"worst err/tol {max(worst):.3f}")


def test_state_and_imu_are_bit_identical_to_the_other_steps():
    """the state of the joint-force step equals the plain step's (no IMU, no effort DOF), the IMU step's (its IMU input too) and the
    effort step's, bit for bit, at 0, 1 and 3 sub-steps"""
    spec = H.spec_for("quad_attitude")
    _, morphy = morphy_compliant()
    _, gimbal = gimbal_quad()
    tg = with_modes(gimbal, "effort")
    for steps in (0, 1, 3):
        inp = _limit_crossing(substep_inputs(spec, morphy, 32, 20 + steps), morphy)
        plain = CpuArticulatedHp1Engine(spec, 32, per_env_params="all", articulation=morphy)
        load_inputs(plain, inp)
        plain.physics_step(inp["actions"], disturbance=inp["dist"], physics_steps=steps)
        jf = run_jf(spec, morphy, inp, physics_steps=steps)
        imu = CpuImuHp1Engine(spec, 32, per_env_params="all", articulation=morphy, imu_body=4)
        load_inputs(imu, inp)
        imu.physics_step(inp["actions"], disturbance=inp["dist"], physics_steps=steps)
        jfi = run_jf(spec, morphy, inp, physics_steps=steps, imu_body=4)
        for k in STATE:
            assert torch.equal(getattr(plain, k), getattr(jf, k)), (steps, k)
            assert torch.equal(getattr(imu, k), getattr(jfi, k)), (steps, k)
        assert torch.equal(imu.imu_input, jfi.imu_input), steps
        assert torch.equal(jf.joint_wrench, jfi.joint_wrench) and torch.equal(jf.dof_force, jfi.dof_force)
        inp = _limit_crossing(substep_inputs(spec, tg, 32, 30 + steps), tg)
        e = effort_inputs(tg, 32, 31)
        eff = CpuEffortHp1Engine(spec, 32, per_env_params="all", articulation=tg, imu_body=2)
        load_inputs(eff, inp)
        eff.dof_actuation_force.copy_(e)
        eff.physics_step(inp["actions"], disturbance=inp["dist"], physics_steps=steps)
        jfe = run_jf(spec, tg, inp, physics_steps=steps, imu_body=2, effort=e)
        for k in STATE + ("imu_input",):
            assert torch.equal(getattr(eff, k), getattr(jfe, k)), (steps, k)
        if steps == 0:
            assert (jfe.joint_wrench == 0).all() and (jfe.dof_force == 0).all()


def test_last_substep_start():
    """a 3-sub-step launch writes the joint forces of its last sub-step: those of a 1-sub-step launch from the state after 2 plain
    sub-steps, bit for bit"""
    spec = H.spec_for("quad_attitude")
    _, art = morphy_compliant()
    inp = _limit_crossing(substep_inputs(spec, art, 32, 11), art)
    three = run_jf(spec, art, inp, physics_steps=3)
    two = CpuArticulatedHp1Engine(spec, 32, per_env_params="all", articulation=art)
    load_inputs(two, inp)
    two.physics_step(inp["actions"], disturbance=inp["dist"], physics_steps=2)
    one = CpuJointForceHp1Engine(spec, 32, per_env_params="all", articulation=art, joint_force=True)
    for k in ("root_state", "motor_thrust", "dof_state", "dof_position_setpoint", "dof_velocity_setpoint", "tau_inc", "tau_dec", "k_thrust",
              "K_pos", "K_vel", "K_rot", "K_angvel"):
        getattr(one, k).copy_(getattr(two, k))
    one.physics_step(inp["actions"], disturbance=inp["dist"], physics_steps=1)
    assert torch.equal(three.joint_wrench, one.joint_wrench) and torch.equal(three.dof_force, one.dof_force)


def test_clamp_ten_times_the_limit_gives_the_same_outputs():
    spec = H.spec_for("quad_attitude")
    _, art = gimbal_quad()
    art = with_modes(art, "effort")
    E = torch.tensor(art.effort_limit, dtype=torch.float32)
    inp = substep_inputs(spec, art, 16, 3)
    sign = torch.where(torch.arange(16)[:, None] % 2 == 0, 1.0, -1.0)
    a = run_jf(spec, art, inp, physics_steps=3, effort=sign * E)
    b = run_jf(spec, art, inp, physics_steps=3, effort=sign * 10 * E)
    for k in ("root_state", "dof_state", "joint_wrench", "dof_force"):
        assert torch.equal(getattr(a, k), getattr(b, k)), k


# ---- physics ------------------------------------------------------------------------------------------------------------------
def _env(robot, env_name="empty_env", n=4, **args):
    from aerial_gym_simulator_b200.env_manager.env_manager import EnvManager
    return EnvManager("base_sim", env_name, robot, "lee_attitude_control", "cpu", num_envs=n, args={"seed": 1, **args})


def _register(name, base):
    from aerial_gym_simulator_b200.registry._core import robot_registry
    from aerial_gym_simulator_b200.robots import ArticulatedMultirotor, BaseMultirotor

    class Cfg(base):
        class joint_config(getattr(base, "joint_config", object)):
            enable_dof_force_sensors = True
    robot_registry.register(name, ArticulatedMultirotor if hasattr(base, "joint_config") else BaseMultirotor, Cfg)
    return name


def _hover(robot, n=8, steps=300):
    env = _env(robot, n=n)
    env.spec.enable_disturbance = False
    env.reset()
    gtd = env.global_tensor_dict
    gtd["dof_state_tensor"].zero_()
    st = gtd["robot_state_tensor"]
    st[:, 3:13] = 0.0
    st[:, 6] = 1.0
    for _ in range(steps):
        env.step(torch.zeros(n, 4))
    return env, gtd


def test_hovering_morphy_flap_joints_carry_the_static_load():
    """hovering morphy_compliant: each flap joint holds its motor's thrust less the motor body's weight on the 0.07 m arm from the
    hinge, (f - m_motor g) 0.07 m, within 5 % (the flap's deflection and the base's residual motion).  Its sign is that of the torque
    the hinge must apply to hold the arm: -axis . (r x z) (f - m_motor g), r the motor's offset from the hinge and z the world's up
    axis, both in the flap body's frame"""
    from aerial_gym_simulator_b200.config import robot_config as rc
    name = _register("_test_morphy_jf", rc.MorphyCompliantCfg)
    with joint_force_cpu_stack():
        torch.manual_seed(0)
        env, gtd = _hover(name)
        b = env.robot.bodies
        f = gtd["dof_force_tensor"].double()
        thrust = env.engine.motor_thrust.double()
        rows = gtd["robot_body_state_tensor"].double()
        for arm in range(4):
            flap = 2 + 2 * arm
            motor = int(env.engine.articulation.motor_body.tolist().index(flap))
            r = torch.tensor(b.com[flap], dtype=torch.float64)
            assert abs(float(r.norm()) - 0.07) < 1e-9
            z = HO.quat_rotate_inverse(rows[:, flap, 3:7], torch.tensor([0.0, 0.0, 1.0], dtype=torch.float64).expand(len(f), 3))
            sign = -(torch.cross(r.expand_as(z), z, dim=1) @ torch.tensor(b.axis[flap], dtype=torch.float64)) / 0.07
            load = (thrust[:, motor] - float(b.mass[flap]) * 9.81) * 0.07
            assert (load > 0.01).all() and (sign.abs() > 0.95).all()
            err = (f[:, flap - 1] - sign * load).abs() / load
            assert err.max() < 0.05, (arm, err)


def test_hovering_gimbal_stages_carry_their_weight_and_no_axis_torque():
    """the gimbal quad at hover: the roll stage's joint carries the weight of both stages, (m_roll + m_pitch) g, the pitch stage's
    carries m_pitch g (its camera link merged in), and each stage is balanced on its axis, so the torque along it is ~0 against the
    stage's weight times its 6 cm drop"""
    from aerial_gym_simulator_b200.config import robot_config as rc
    name = _register("_test_gimbal_jf", rc.BaseQuadWithGimbalCameraCfg)
    with joint_force_cpu_stack():
        torch.manual_seed(0)
        env, gtd = _hover(name)
        b = env.robot.bodies
        W = gtd["robot_joint_wrench_tensor"].double()
        assert gtd["robot_body_names"] == ["base_link", "roll_stage_link", "pitch_stage_link"]
        m1, m2 = float(b.mass[1]), float(b.mass[2])
        g = 9.81
        np.testing.assert_allclose(W[:, 1, 0:3].norm(dim=1).numpy(), (m1 + m2) * g, rtol=0.02)
        np.testing.assert_allclose(W[:, 2, 0:3].norm(dim=1).numpy(), m2 * g, rtol=0.02)
        f = gtd["dof_force_tensor"].double()
        assert f.abs().max() < 0.02 * (m1 + m2) * g * 0.06, f


# ---- host layer ----------------------------------------------------------------------------------------------------------------
def test_env_publishes_the_tensors_only_with_the_flag():
    from aerial_gym_simulator_b200.config import robot_config as rc
    names = [_register("_test_gimbal_jf2", rc.BaseQuadWithGimbalCameraCfg), _register("_test_torque_gimbal_jf", rc.BaseQuadWithTorqueGimbalCfg)]
    with joint_force_cpu_stack():
        for robot in names:
            torch.manual_seed(0)
            env = _env(robot)
            gtd, eng = env.global_tensor_dict, env.engine
            assert gtd["dof_force_tensor"] is eng.dof_force and gtd["dof_force_tensor"].shape == (4, 2)
            assert gtd["robot_joint_wrench_tensor"] is eng.joint_wrench and eng.joint_wrench.shape == (4, 3, 6)
            assert (eng.joint_wrench == 0).all() and (eng.dof_force == 0).all()
            env.reset()
            env.step(torch.zeros(4, 4))
            assert (eng.joint_wrench[:, 1:] != 0).any() and (eng.joint_wrench[:, 0] == 0).all()
            before = eng.joint_wrench.clone()
            env.reset_idx(torch.tensor([0, 2]))
            assert torch.equal(eng.joint_wrench, before)  # a reset leaves them as the last step wrote them
        for robot in ("base_quadrotor_with_gimbal_camera", "morphy_compliant", "base_quadrotor_with_torque_gimbal"):
            env = _env(robot)
            assert "dof_force_tensor" not in env.global_tensor_dict and "robot_joint_wrench_tensor" not in env.global_tensor_dict
            assert env.engine.joint_wrench is None and env.engine.dof_force is None


def test_rigid_robot_raises():
    from aerial_gym_simulator_b200.config import robot_config as rc
    name = _register("_test_quad_jf", rc.BaseQuadCfg)
    with joint_force_cpu_stack():
        with pytest.raises(ValueError, match="joint_force belongs to an articulated robot"):
            _env(name)


def test_c_abi_validation():
    lib = _lib.load()
    spec = H.spec_for("quad_attitude")
    _, art = gimbal_quad()
    tg = with_modes(art, "effort")
    buf, s, e = _lib.AgxHp1Buffers(), tg.to_struct(), tg.effort_struct()
    jw, df, imu = torch.zeros(64, 3, 6), torch.zeros(64, 2), torch.zeros(64, 9)
    call = lambda n, eff, b=0, im=None, w=jw.data_ptr(), d=df.data_ptr(), st=s: lib.agx_hp1_articulated_step_joint_force(
        C.byref(build_config(spec, n)), C.byref(buf), C.byref(st), eff, b, im, w, d, None)
    assert call(0, C.byref(e)) == 0 and call(0, None, 2, imu.data_ptr()) == 0 and call(0, None, w=None, d=None) == 0
    assert call(0, C.byref(e), 3, imu.data_ptr()) != 0 and b"imu_body" in lib.agx_last_error()
    e2 = tg.effort_struct()
    e2.effort_limit[1] = -0.1
    assert call(0, C.byref(e2)) != 0 and b"effort_limit[1]" in lib.agx_last_error()
    s2 = tg.to_struct()
    s2.stiffness[2] = 0.5
    assert call(0, C.byref(e), st=s2) != 0 and b"stiffness[2]" in lib.agx_last_error()
    # one env with non-NULL state buffers: the outputs are checked before any launch
    x = torch.zeros(64)
    buf.root_state, buf.motor_thrust, buf.actions = x.data_ptr(), x.data_ptr(), x.data_ptr()
    s.dof_state = s.dof_position_setpoint = s.dof_velocity_setpoint = x.data_ptr()
    assert call(1, C.byref(e)) != 0 and b"effort->effort is NULL" in lib.agx_last_error()
    e.effort = x.data_ptr()
    for w, d in ((None, df.data_ptr()), (jw.data_ptr(), None)):
        assert call(1, C.byref(e), w=w, d=d) != 0 and b"joint_wrench/dof_force is NULL" in lib.agx_last_error()
    for w, d in ((jw.data_ptr() + 8, df.data_ptr()), (jw.data_ptr(), df.data_ptr() + 4)):
        assert call(1, C.byref(e), w=w, d=d) != 0 and b"16-byte aligned" in lib.agx_last_error()


# ---- machine code ----------------------------------------------------------------------------------------------------------------
# -Xptxas -v of the four instantiations of articulated_step_joint_force_kernel<M, NB> (CUDA 12.9, sm_90a): registers per thread.  The
# stack frame is the per-body arrays of the ABA, in local memory by design (articulated.cu), the same as articulated_step_kernel's.
JF_KERNEL_REGS = {(4, 9): 165, (4, 16): 165, (8, 9): 168, (8, 16): 168}
JF_KERNEL_STACK = {9: 3312, 16: 5856}
# normalised SASS (test_articulated_imu_cpu.sass_functions), md5, of every kernel articulated.cu had before the joint-force entry point
PARENT_SASS = {
    "articulated_step_kernelILi4ELi16E": "61f12510a9b31d109fae04dc1a814d87",
    "articulated_step_kernelILi4ELi9E": "efbd4a3c22e2ad0447001440b6c8ac27",
    "articulated_step_kernelILi8ELi16E": "4d833f5c266d542fe19e29d2b82ef233",
    "articulated_step_kernelILi8ELi9E": "c2086c00bb11078baa2a0b9cc19015ce",
    "articulated_step_imu_kernelILi4ELi16E": "126c2d9df2119902e827c3866d83e9fb",
    "articulated_step_imu_kernelILi4ELi9E": "2b321c922eed32aa91bc91d3594f5433",
    "articulated_step_imu_kernelILi8ELi16E": "f4eb229df3dcb4a243ca0d7daecea392",
    "articulated_step_imu_kernelILi8ELi9E": "8418465ed540f9c3753c25a8ffefbfff",
    "articulated_step_effort_kernelILi4ELi16ELb0E": "09c0d3e7332544ce33a23224720c7ea1",
    "articulated_step_effort_kernelILi4ELi16ELb1E": "9579cc186f99b4fd0882a770a5f271e5",
    "articulated_step_effort_kernelILi4ELi9ELb0E": "abd31654971564ffba13ba49beb4fec6",
    "articulated_step_effort_kernelILi4ELi9ELb1E": "f6b6f80c1bcce608057bcdea4b8ec6cb",
    "articulated_step_effort_kernelILi8ELi16ELb0E": "3460f725d21829e0b968c1d33a994119",
    "articulated_step_effort_kernelILi8ELi16ELb1E": "1574c81ff97a7ac7fc0231afe3a3f2a2",
    "articulated_step_effort_kernelILi8ELi9ELb0E": "c3c8b9d43a5e98e00d872969082d91ee",
    "articulated_step_effort_kernelILi8ELi9ELb1E": "a32e11ab74110bf4d33d9e436db96c31",
    "articulated_body_state_kernelILi16E": "49fabc56648bbeedb676825c9dfce8b7",
    "articulated_body_state_kernelILi9E": "d6ab5ca7ca0215f6f63b3496123fa2d8",
}


def test_joint_force_kernels_have_no_spills(articulated_unit):  # noqa: F811
    log, _ = articulated_unit
    blocks = re.findall(r"Compiling entry function '(\S+)'.*?\n.*?(\d+) bytes stack frame, (.*?spill loads)\n.*?Used (\d+) registers", log,
                        re.S)
    found = {}
    for f, stack, info, regs in blocks:
        m = re.search(r"articulated_step_joint_force_kernelILi(\d)ELi(\d+)E", f)
        if m:
            assert info == "0 bytes spill stores, 0 bytes spill loads", (f, info)
            assert int(stack) == JF_KERNEL_STACK[int(m.group(2))], (f, stack)
            found[(int(m.group(1)), int(m.group(2)))] = int(regs)
    assert found == JF_KERNEL_REGS, found


def test_pre_existing_kernels_keep_their_sass(articulated_unit):  # noqa: F811
    _, sass = articulated_unit
    h = sass_functions(sass)
    for key, md5 in PARENT_SASS.items():
        hits = [v for k, v in h.items() if key in k]
        assert hits == [md5], (key, hits)
