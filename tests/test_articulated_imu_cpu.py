"""The IMU on a link of an articulated robot, on the CPU (DESIGN.md "Articulated robots", "IMU on a link"): the IMU input of
art_env_step<M, NB, true> (host shadow, tests/csrc/articulated_imu_shadow.cu) against oracle/articulated_imu_oracle.py, the oracle
itself against central differences, momentum balance and the rigid path, and the host layer (EnvManager, IMUSensor) on the CPU stack."""
import ctypes as C
import hashlib
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from aerial_gym_simulator_b200 import _build, _lib
from oracle import articulated_body_state_oracle as BO
from oracle import articulated_imu_oracle as IO
from oracle import articulated_oracle as AO
from oracle import aux_oracle as XO
from oracle import hp1_oracle as HO

from . import _hp1_common as H
from ._cpu_stack_articulated import CpuArticulatedHp1Engine
from ._cpu_stack_articulated_imu import CpuImuHp1Engine, imu_cpu_stack
from .test_articulated_body_state_cpu import gimbal_levelling
from .test_articulated_cpu import RTOL, load_inputs, morphy_compliant, oracle_state, random_art, random_root, shaped_art, \
    substep_inputs, table_of

EPS = float(np.finfo(np.float32).eps)
ULPS = 8


def gimbal_quad():
    import aerial_gym_simulator_b200.robots  # noqa: F401
    from aerial_gym_simulator_b200.config.env_config import EmptyEnvCfg
    from aerial_gym_simulator_b200.registry._core import robot_registry
    robot, _ = robot_registry.make_robot("base_quadrotor_with_gimbal_camera", "lee_attitude_control", EmptyEnvCfg, "cpu")
    return robot, robot.make_articulation()


def _depth(table, b):
    d = 0
    while b > 0:
        b, d = int(table["parent"][b]), d + 1
    return d


# ---- the IMU input against the float64 oracle --------------------------------------------------------------------------------
# Tolerance of (f, n, w_b) of body b (depth d below the base).  The float32 ABA gives a0 and every qdd within RTOL amax of the
# float64 solve (amax = max |(a0, qdd)| of the env; test_articulated_cpu.py section 2); body b's spatial acceleration sums d + 1 such
# terms, each times a motion subspace whose linear part is a lever arm of at most L = the largest |P_i| + |c| of the tree, so
# E_ang = RTOL amax (d + 1) and E_lin = E_ang (1 + L); the COM acceleration adds E_ang |c| to E_lin.  The rotation R_b is off by
# e_R = 32 eps (d + 1) (the bar of test_articulated_body_state_cpu.py), which turns each vector by that much; every product and sum
# adds ULPS ulps of its magnitude.  So, with a the magnitude of the terms of a_c - g (|a^| + |alpha| |c| + |w| (|v_O| + |w| |c|) + |g|):
#   f:   m (E_lin + E_ang |c|) + m (e_R + ULPS eps) a
#   n:   |I| E_ang + |I| (e_R + ULPS eps) (|alpha| + |w|^2)
#   w_b: (e_R + ULPS eps) |w| + ULPS eps (|w_0| + Q), Q = the sum of |q-dot| along the path.
def imu_tolerance(table, b, root, q, qd, a0, qdd, grav):
    R, P, V, A = IO.body_motion(table, root, q, qd, a0, qdd)
    c, _ = IO.com_acceleration(table, b, R, P, V, A)
    d = _depth(table, b)
    L = max(float(np.linalg.norm(P[i] + R[i] @ table["com"][i])) for i in range(int(table["num_bodies"])))
    amax = float(np.abs(np.concatenate([a0, qdd])).max())
    e_ang = RTOL * amax * (d + 1)
    e_lin = e_ang * (1.0 + L)
    eR = 32 * EPS * (d + 1)
    w, al = np.linalg.norm(V[b, :3]), np.linalg.norm(A[b, :3])
    cn = np.linalg.norm(c)
    a = np.linalg.norm(A[b, 3:]) + al * cn + w * (np.linalg.norm(V[b, 3:]) + w * cn) + np.linalg.norm(grav)
    m, In = float(table["mass"][b]), float(np.abs(table["inertia"][b]).sum())
    path = []
    k = b
    while k > 0:
        path.append(k)
        k = int(table["parent"][k])
    Q = sum(abs(float(qd[k - 1])) for k in path)
    tf = m * (e_lin + e_ang * cn) + m * (eR + ULPS * EPS) * a
    tn = In * e_ang + In * (eR + ULPS * EPS) * (al + w * w)
    tw = (eR + ULPS * EPS) * w + ULPS * EPS * (np.linalg.norm(root[10:13]) + Q)
    return np.array([tf] * 3 + [tn] * 3 + [tw] * 3)


def run_shadow(spec, art, b, inp, physics_steps=1):
    n = inp["root"].shape[0]
    eng = CpuImuHp1Engine(spec, n, per_env_params="all", articulation=art, imu_body=b)
    load_inputs(eng, inp)
    eng.physics_step(inp["actions"], disturbance=inp["dist"], physics_steps=physics_steps)
    return eng


def check_imu(eng, spec, inp, b, idx, got=None, worst=None):
    """the engine's imu_input (or `got`) of envs idx against IO.substep_imu at the inputs' state, with imu_tolerance; envs that fail
    _hp1_common.well_conditioned are only checked for finite values.  -> worst err / tol"""
    model, st = oracle_state(eng, spec, inp, idx)
    ok = H.well_conditioned(model, st, inp["actions"][idx].double()).numpy()
    dof = inp["dof"][idx].double().numpy()
    table = table_of(eng.art)
    ref, ex = IO.substep_imu(model, table, st, dof[..., 0], dof[..., 1], inp["qs"][idx].double().numpy(), inp["qds"][idx].double().numpy(),
                             inp["actions"][idx].double(), b, inp["dist"][idx].double())
    got = (eng.imu_input if got is None else got).detach().cpu().double().numpy()[idx]
    assert np.isfinite(got).all()
    r = 0.0
    for k in np.flatnonzero(ok):
        tol = imu_tolerance(table, b, st.root[k].numpy(), dof[k, :, 0], dof[k, :, 1], ex["a0"][k], ex["qdd"][k], model.gravity)
        err = np.abs(got[k] - ref[k])
        assert (err <= tol).all(), (k, err, tol)
        r = max(r, float(np.max(err / np.where(tol > 0, tol, 1.0))))
    if worst is not None:
        worst.append(r)
    return r, ok


def _limit_crossing(inp, art):
    """joints started at their limits with velocities pointing out of the range: the sub-step projects them"""
    b = art.bodies
    lim = np.flatnonzero(b.limited[1:])
    if lim.size:
        dof = inp["dof"].numpy()
        side = np.where(np.arange(dof.shape[0]) % 2 == 0, 1.0, -1.0)[:, None]
        dof[:, lim, 0] = np.where(side > 0, b.upper[1:][lim], b.lower[1:][lim]).astype(np.float32)
        dof[:, lim, 1] = (side * 2.0).astype(np.float32)
        inp["dof"] = torch.from_numpy(dof)
    return inp


@pytest.mark.parametrize("robot", ["morphy_compliant", "gimbal"])
def test_shadow_matches_oracle_on_shipped_robots(robot):
    """imu_body = the base, a middle body and a leaf; drives on (the robot's own gains) and off; joints inside and crossing limits"""
    spec = H.spec_for("quad_attitude")
    _, art = morphy_compliant() if robot == "morphy_compliant" else gimbal_quad()
    B = art.bodies.num_bodies
    bodies = (0, 1, B - 1) if robot == "gimbal" else (0, 1, 8)
    worst = []
    for drive in (True, False):
        if not drive:
            art.stiffness[:] = 0.0
            art.damping[:] = 1e-4  # the massless connecting links of morphy need some drive for a defined acceleration
        for b in bodies:
            if not art.bodies.mass[b] > 0:
                continue
            for cross in (False, True):
                inp = substep_inputs(spec, art, 24, 300 + b + 10 * cross + 20 * drive)
                if cross:
                    inp = _limit_crossing(inp, art)
                eng = run_shadow(spec, art, b, inp)
                check_imu(eng, spec, inp, b, np.arange(24), worst=worst)
    print(f"worst err/tol {max(worst):.3f}")


@pytest.mark.parametrize("M", [4, 8])
def test_shadow_matches_oracle_on_random_trees(M):
    rng = np.random.default_rng(60 + M)
    spec = H.spec_for("quad_attitude" if M == 4 else "octa_velocity")
    worst = []
    for B in range(1, 17):
        art = shaped_art(rng, B, M=M, drive=bool(B % 2))
        for b in sorted({0, B // 2, B - 1}):
            inp = substep_inputs(spec, art, 16, 500 + 17 * B + b)
            eng = run_shadow(spec, art, b, inp)
            check_imu(eng, spec, inp, b, np.arange(16), worst=worst)
    print(f"worst err/tol {max(worst):.3f}")


def test_state_outputs_are_bit_identical_to_the_plain_step():
    spec = H.spec_for("quad_attitude")
    _, art = morphy_compliant()
    for steps in (0, 1, 3):
        inp = _limit_crossing(substep_inputs(spec, art, 32, 9), art)
        plain = CpuArticulatedHp1Engine(spec, 32, per_env_params="all", articulation=art)
        load_inputs(plain, inp)
        plain.physics_step(inp["actions"], disturbance=inp["dist"], physics_steps=steps)
        imu = run_shadow(spec, art, 4, inp, physics_steps=steps)
        for k in ("root_state", "motor_thrust", "dof_state") + CpuArticulatedHp1Engine.DERIVED:
            assert torch.equal(getattr(plain, k), getattr(imu, k)), (steps, k)


def test_last_substep_start_and_zero_steps():
    """a 3-sub-step launch writes the IMU input of its last sub-step: that of a 1-sub-step launch from the state after 2 plain
    sub-steps, bit for bit.  With physics_steps = 0: f = n = 0 and w_b of the unstepped state."""
    spec = H.spec_for("quad_attitude")
    _, art = morphy_compliant()
    inp = _limit_crossing(substep_inputs(spec, art, 32, 11), art)
    three = run_shadow(spec, art, 2, inp, physics_steps=3)
    two = CpuArticulatedHp1Engine(spec, 32, per_env_params="all", articulation=art)
    load_inputs(two, inp)
    two.physics_step(inp["actions"], disturbance=inp["dist"], physics_steps=2)
    one = CpuImuHp1Engine(spec, 32, per_env_params="all", articulation=art, imu_body=2)
    for k in ("root_state", "motor_thrust", "dof_state", "dof_position_setpoint", "dof_velocity_setpoint", "tau_inc", "tau_dec", "k_thrust",
              "K_pos", "K_vel", "K_rot", "K_angvel"):
        getattr(one, k).copy_(getattr(two, k))
    one.physics_step(inp["actions"], disturbance=inp["dist"], physics_steps=1)
    assert torch.equal(three.imu_input, one.imu_input)
    zero = run_shadow(spec, art, 6, inp, physics_steps=0)
    assert (zero.imu_input[:, 0:6] == 0).all()
    table = table_of(zero.art)
    for n in range(32):
        r = inp["root"][n].double().numpy()
        dof = inp["dof"][n].double().numpy()
        R, P, V, A = IO.body_motion(table, r, dof[:, 0], dof[:, 1], np.zeros(6), np.zeros(8))
        np.testing.assert_allclose(zero.imu_input[n, 6:9].double().numpy(), R[6].T @ V[6, :3], atol=1e-5)


# ---- the oracle itself ---------------------------------------------------------------------------------------------------------
def _random_case(rng, B, M=4):
    art = random_art(rng, B, M=M)
    table = table_of(art.to_struct())
    D = B - 1
    root = random_root(rng)
    return art, table, root, rng.uniform(-1, 1, D), rng.uniform(-2, 2, D), rng.uniform(-1, 1, D), rng.uniform(-1, 1, D), \
        rng.uniform(0, 2, M), rng.uniform(-1, 1, 3), rng.uniform(-0.05, 0.05, 3)


def test_oracle_com_acceleration_is_the_derivative_of_the_com_velocity():
    """central differences of each body's COM velocity (from body_states) along the ABA accelerations"""
    rng = np.random.default_rng(3)
    h = 1e-5
    grav = np.array([0.0, 0.0, -9.81])
    for B in (1, 2, 9, 16):
        _, table, root, q, qd, qs, qds, th, F, T = _random_case(rng, B)
        a0, qdd = AO.dynamics(table, root, q, qd, qs, qds, 0.01, grav, th, F, T)
        R, P, V, A = IO.body_motion(table, root, q, qd, a0, qdd)
        w, v = root[10:13], root[7:10]

        def com_vel(t):
            r = root.copy()
            wt = w + a0[:3] * t
            th_ = w * t + 0.5 * a0[:3] * t * t  # rotation vector to second order (for a velocity that changes linearly)
            ang = np.linalg.norm(th_)
            Rw = AO._rot(th_ / ang, ang) if ang > 0 else np.eye(3)
            r[0:3] = root[0:3] + v * t
            r[3:7] = BO.matrix_to_quat(Rw @ AO.quat_to_matrix(root[3:7]))
            r[7:10] = v + (a0[3:] + np.cross(w, v)) * t
            r[10:13] = wt
            rows = BO.body_states(table, r, q + qd * t + 0.5 * qdd * t * t, qd + qdd * t)
            out = []
            for i in range(B):
                Ri = AO.quat_to_matrix(rows[i, 3:7])
                out.append(rows[i, 7:10] + np.cross(rows[i, 10:13], Ri @ table["com"][i]))
            return np.array(out)
        fd = (com_vel(h) - com_vel(-h)) / (2 * h)
        for i in range(B):
            _, ac = IO.com_acceleration(table, i, R, P, V, A)
            assert np.abs(fd[i] - ac).max() < 1e-4 * (1 + np.abs(ac).max()), (B, i, fd[i], ac)


def test_oracle_momentum_balance():
    """sum_b R_b f_b = the world sum of the thrusts, drag and disturbance: the joint reactions cancel pairwise"""
    rng = np.random.default_rng(4)
    grav = np.array([0.0, 0.0, -9.81])
    cases = [(morphy_compliant()[1], None)] + [(None, B) for B in range(1, 17)]
    for art, B in cases:
        for _ in range(4):
            if art is None:
                a, table, root, q, qd, qs, qds, th, F, T = _random_case(rng, B)
            else:
                a, table = art, table_of(art.to_struct())
                D = a.num_dofs
                root, q, qd, qs, qds = random_root(rng), rng.uniform(-0.5, 0.5, D), rng.uniform(-2, 2, D), rng.uniform(-1, 1, D), \
                    rng.uniform(-1, 1, D)
                th, F, T = rng.uniform(0, 2, 4), rng.uniform(-1, 1, 3), rng.uniform(-0.05, 0.05, 3)
            a0, qdd = AO.dynamics(table, root, q, qd, qs, qds, 0.01, grav, th, F, T)
            R, P, V, A = IO.body_motion(table, root, q, qd, a0, qdd)
            total, tol = np.zeros(3), 1e-9 * (1 + np.abs(F).max() + np.abs(th).sum())
            for b in range(int(table["num_bodies"])):
                u = IO.imu_from_motion(table, b, grav, R, P, V, A)
                total += R[b] @ u[0:3]
                # the table's rotations are float32 roundings, orthonormal only to ~1e-7: R_b R_b^T f moves by that defect
                tol += np.abs(R[b] @ R[b].T - np.eye(3)).sum() * np.abs(u[0:3]).max()
            ext = F.copy()
            for k in range(len(th)):
                ext += (R[int(table["motor_body"][k])] @ table["motor_R"][k])[:, 2] * th[k]
            assert np.abs(total - ext).max() <= tol, (total, ext, tol)


def test_oracle_one_body_tree_is_the_rigid_path():
    """one body, its COM at the origin, the HP1 model's mass and inertia: f_0, n_0 and w_0 are hp1_oracle's F_body, T_body and the
    derived body_angvel of the sub-step's start, to rounding"""
    n = 128
    spec = H.spec_for("quad_attitude")
    spec.drag_lin1, spec.drag_ang1 = (0.1, 0.1, 0.2), (1e-3,) * 3
    model = H.oracle_model_from_spec(spec)
    z1 = np.zeros(1)
    tab = {"num_bodies": 1, "parent": np.array([-1]), "joint_R": np.eye(3)[None], "joint_p": np.zeros((1, 3)), "axis": np.zeros((1, 3)),
           "mass": np.array([model.mass]), "com": np.zeros((1, 3)), "inertia": model.inertia[None], "stiffness": z1, "damping": z1,
           "motor_body": np.zeros(4, int), "motor_R": model.link_R, "motor_p": model.link_r,
           "motor_torque": -model.thrust_to_torque_ratio * model.motor_directions, "lower": z1, "upper": z1, "limited": z1}
    root, actions, params = H.random_inputs(spec, n, 23)
    st = H.load_oracle_state(model, root.double(), {k: v.double() for k, v in params.items()}, n)
    st.root[:, 3:7] /= st.root[:, 3:7].norm(dim=1, keepdim=True)
    dist = torch.rand(n, 6, dtype=torch.float64, generator=torch.Generator().manual_seed(5)) - 0.5
    z = np.zeros((n, 0))
    u, _ = IO.substep_imu(model, tab, st.clone(), z, z, z, z, actions.double(), 0, dist)
    st1 = st.clone()
    out = HO.physics_step(model, st1, actions.double(), dist)
    F, T = out["F_body"].numpy(), out["T_body"].numpy()
    np.testing.assert_allclose(u[:, 0:3], F, rtol=0, atol=1e-9 * (1 + np.abs(F).max()))
    np.testing.assert_allclose(u[:, 3:6], T, rtol=0, atol=1e-9 * (1 + np.abs(T).max()))
    np.testing.assert_allclose(u[:, 6:9], st1.derived["body_angvel"].numpy(), rtol=0, atol=1e-12)


# ---- the host layer --------------------------------------------------------------------------------------------------------------
def _env(robot, env_name="empty_env", n=8, **args):
    from aerial_gym_simulator_b200.env_manager.env_manager import EnvManager
    return EnvManager("base_sim", env_name, robot, "lee_attitude_control", "cpu", num_envs=n, args=args or None)


def _imu_cfg(base, link, **kw):
    class Imu(base.sensor_config.imu_config):
        parent_link = link
    for k, v in kw.items():
        setattr(Imu, k, v)
    return Imu


def _register(name, base, link, **kw):
    from aerial_gym_simulator_b200.registry._core import robot_registry
    from aerial_gym_simulator_b200.robots import ArticulatedMultirotor, BaseMultirotor
    imu = _imu_cfg(base, link, **kw) if link is not None else base.sensor_config.imu_config

    class Cfg(base):
        class sensor_config(base.sensor_config):
            enable_imu = True
            imu_config = imu
    robot_registry.register(name, ArticulatedMultirotor if hasattr(base, "joint_config") else BaseMultirotor, Cfg)


@pytest.mark.parametrize("world_frame", [False, True])
def test_measurement_is_imu_update_of_the_oracle_force_input(world_frame):
    """one env step of morphy_compliant with the IMU on a flap's motor body, then render(): imu_measurement equals aux_oracle's
    imu_update on the oracle's force input (f_b of the step's start + m_b R_b,post^T g), R_b,post and w_b, with the same noise and bias
    draws, within the oracle tolerance of f_b / m_b plus the float32 rounding of the IMU's own arithmetic"""
    from aerial_gym_simulator_b200.config import robot_config as rc
    _register(f"_test_morphy_imu_motor_{int(world_frame)}", rc.MorphyCompliantCfg, "arm_motor_0", world_frame=world_frame)
    n = 16
    with imu_cpu_stack():
        torch.manual_seed(0)
        env = _env(f"_test_morphy_imu_motor_{int(world_frame)}", n=n)
        env.spec.enable_disturbance = False
        env.reset()
        gtd, eng = env.global_tensor_dict, env.engine
        b = eng.imu_body
        assert b == env.robot.bodies.link_body["arm_motor_0"] and b > 0
        gtd["dof_position_setpoint_tensor"].fill_(0.2)
        for _ in range(3):
            env.step(torch.rand(n, 4) * 0.4 - 0.2)
        root0, dof0, th0 = eng.root_state.clone(), eng.dof_state.clone(), eng.motor_thrust.clone()
        act = torch.rand(n, 4) * 0.4 - 0.2
        env.step(act)
        torch.manual_seed(7)
        n_noise, n_bias = torch.randn(n, 6), torch.randn(n, 6)
        bias0 = env.imu.bias.clone()
        torch.manual_seed(7)
        env.render()
        meas = gtd["imu_measurement"].double().numpy()
        # the oracle's force input
        inp = {"root": root0, "actions": act, "dist": torch.zeros(n, 6), "dof": dof0,
               "qs": gtd["dof_position_setpoint_tensor"].clone(), "qds": gtd["dof_velocity_setpoint_tensor"].clone(),
               "params": {"thrust": th0, **{k: getattr(eng, k).clone() for k in ("tau_inc", "tau_dec", "k_thrust", "K_pos", "K_vel", "K_rot",
                                                                                  "K_angvel") if getattr(eng, k) is not None}}}
        idx = np.arange(n)
        model, st = oracle_state(eng, env.spec, inp, idx)
        table = table_of(eng.art)
        dof = dof0.double().numpy()
        u, ex = IO.substep_imu(model, table, st, dof[..., 0], dof[..., 1], inp["qs"].double().numpy(), inp["qds"].double().numpy(),
                               act.double(), b, None)
        m = float(table["mass"][b])
        qpost = torch.from_numpy(gtd["robot_body_state_tensor"][:, b, 3:7].double().numpy())
        g = torch.tensor(model.gravity, dtype=torch.float64).expand(n, 3)
        force = torch.from_numpy(u[:, 0:3]) + m * HO.quat_rotate_inverse(qpost, g)
        ic = env.imu.cfg
        ref, _ = XO.imu_update(force, torch.full((n,), m, dtype=torch.float64), qpost, torch.from_numpy(u[:, 6:9]),
                               env.imu.mount_quats.double(), g, world_frame, ic.gravity_compensation, bias0.double(),
                               n_noise.double(), n_bias.double(), torch.tensor(ic.imu_noise_std, dtype=torch.float64),
                               torch.tensor(ic.bias_std, dtype=torch.float64), torch.tensor(ic.max_measurement_value, dtype=torch.float64),
                               env.sim_config.sim.dt, ic.enable_noise, ic.enable_bias)
        for k in range(n):
            tol = imu_tolerance(table, b, st.root[k].numpy(), dof[k, :, 0], dof[k, :, 1], ex["a0"][k], ex["qdd"][k], model.gravity)
            acc_tol = tol[0] / m + 16 * EPS * (np.abs(ref[k, 0:3].numpy()).max() + 9.81)
            gyro_tol = tol[6] + 16 * EPS * np.abs(ref[k, 3:6].numpy()).max()
            assert np.abs(meas[k, 0:3] - ref[k, 0:3].numpy()).max() <= acc_tol
            assert np.abs(meas[k, 3:6] - ref[k, 3:6].numpy()).max() <= gyro_tol


def test_hovering_morphy_reads_gravity_along_body_z():
    """morphy_compliant_imu (IMU on base_link) hovering for 3 s: the accelerometer reads +g along the base's z.  Bound: the noise
    (4 sigma of imu_noise_std / sqrt(dt)), the bias (its initial bound plus 4 sigma of its walk over the run), and what the base's
    residual acceleration can be: the arms still move (|q-ddot| from the last step's change of q-dot) and their reactions on the base
    scale with the arm's lever (the motor 0.07 m beyond the flap hinge, the hinge 0.1 m out) times the arm-to-base mass ratio, and
    the base's tilt, g (1 - cos)"""
    from aerial_gym_simulator_b200.utils.math import quat_mul
    with imu_cpu_stack():
        torch.manual_seed(0)
        env = _env("morphy_compliant_imu", n=16)
        env.spec.enable_disturbance = False
        env.reset()
        gtd = env.global_tensor_dict
        gtd["dof_state_tensor"].zero_()
        st = gtd["robot_state_tensor"]
        st[:, 3:13] = 0.0
        st[:, 6] = 1.0
        steps = 300
        for k in range(steps):
            qd_before = gtd["dof_state_tensor"][..., 1].clone()
            env.step(torch.zeros(16, 4))
        env.render()
        ic = env.imu.cfg
        dt = env.sim_config.sim.dt
        acc = gtd["imu_measurement"][:, 0:3].double()
        qdd = ((gtd["dof_state_tensor"][..., 1] - qd_before).abs().max(1).values / dt).double()
        b = env.robot.bodies
        ratio = float(b.mass[1:].sum() / b.mass[0])
        resid = qdd * 0.17 * ratio
        # +g along the base's z, seen through the sensor's mount (BaseImuConfig draws it within +-2 degrees)
        q_ws = quat_mul(gtd["robot_state_tensor"][:, 3:7].double(), env.imu.mount_quats.double())
        expect = HO.quat_rotate_inverse(q_ws, torch.tensor([0.0, 0.0, 9.81], dtype=torch.float64).expand(16, 3))
        noise = 4 * max(ic.imu_noise_std[0:3]) / np.sqrt(dt)
        bias = max(ic.max_bias_init_value[0:3]) + 4 * max(ic.bias_std[0:3]) * np.sqrt(dt) * np.sqrt(steps)
        bound = noise + bias + resid + 16 * EPS * 9.81
        err = (acc - expect).abs().max(1).values
        assert (err <= bound).all(), (err, bound)
        assert (gtd["dof_state_tensor"][:, 1::2, 0].abs() > 0.01).all()  # the arms do deflect


def test_gimbal_camera_imu_reads_the_specific_force_in_the_levelled_frame():
    """base_quadrotor_with_gimbal_camera_imu commanded to roll 0.3 / pitch -0.2 with levelling targets (DESIGN's gimbal test).  The
    specific force of a banked multirotor is its thrust over its mass, along the base's z axis: a base_link IMU reads it along its own
    z, while the levelled camera link -- whose z stays vertical within the levelling bound -- reads it tilted by the base's roll and
    pitch.  The camera IMU's gyro reads a link at rest in the world's yaw frame."""
    from aerial_gym_simulator_b200.config import robot_config as rc
    exact = dict(enable_noise=False, enable_bias=False, min_euler_rotation_deg=[0.0] * 3, max_euler_rotation_deg=[0.0] * 3)
    _register("_test_gimbal_base_imu", rc.BaseQuadWithGimbalCameraCfg, "base_link", **exact)
    _register("_test_gimbal_cam_imu", rc.BaseQuadWithGimbalCameraImuCfg, "gimbal_camera_link", **exact)
    out = {}
    with imu_cpu_stack():
        for name in ("_test_gimbal_base_imu", "_test_gimbal_cam_imu"):
            torch.manual_seed(0)
            env = _env(name, n=4)
            x, e = gimbal_levelling(env, 100, "cpu")
            env.render()
            out[name] = (env.global_tensor_dict["imu_measurement"].double().clone(), e)
    acc_b, e = out["_test_gimbal_base_imu"][0][:, 0:3], out["_test_gimbal_base_imu"][1]
    acc_c, gyro_c = out["_test_gimbal_cam_imu"][0][:, 0:3], out["_test_gimbal_cam_imu"][0][:, 3:6]
    LEVEL = 5e-3  # test_articulated_body_state_cpu.LEVEL_TOL
    # base: along its z (the thrust axis)
    assert (acc_b[:, 0:2].norm(dim=1) / acc_b.norm(dim=1)).max() < 2 * LEVEL
    # camera: the same magnitude, tilted by the base's attitude: its angle to the camera's z is the base's tilt
    tilt = torch.acos(torch.cos(e[:, 0]) * torch.cos(e[:, 1]))
    ang = torch.acos(acc_c[:, 2] / acc_c.norm(dim=1))
    assert (ang - tilt).abs().max() < 4 * LEVEL, (ang, tilt)
    assert ((acc_c.norm(dim=1) - acc_b.norm(dim=1)).abs() / acc_b.norm(dim=1)).max() < 1e-2
    assert gyro_c.abs().max() < 0.05


def test_parent_link_on_a_rigid_robot_only_folds_the_orientation():
    """a rigid robot's IMU on motor_0 (a link with the root's orientation): the same reading as today's base IMU, bit for bit; the
    sensor reads robot_state_tensor, robot_mass and body_wrench as before, with mount_quats = q_l (x) sensor_quats"""
    from aerial_gym_simulator_b200.config import robot_config as rc
    _register("_test_quad_imu_motor", rc.BaseQuadWithImuCfg, "motor_0")
    meas = {}
    with imu_cpu_stack():
        for name in ("base_quadrotor_with_imu", "_test_quad_imu_motor"):
            torch.manual_seed(0)
            env = _env(name, n=8)
            env.reset()
            for _ in range(3):
                env.step(torch.rand(8, 4) * 0.2)
                env.reset_idx(torch.tensor([2]))
                env.render()
            meas[name] = env.global_tensor_dict["imu_measurement"].clone()
            if name == "_test_quad_imu_motor":
                assert env.imu.robot_state is env.global_tensor_dict["robot_state_tensor"]
                assert env.engine.imu_input is None and env.engine.body_wrench is not None
                assert torch.equal(env.imu.mount_quats, env.imu.sensor_quats)
            else:
                assert env.imu.mount_quats is env.imu.sensor_quats and env.imu.link_quat is None
    assert torch.equal(meas["base_quadrotor_with_imu"], meas["_test_quad_imu_motor"])


def test_link_fold_after_every_draw():
    from aerial_gym_simulator_b200.utils.math import quat_mul
    with imu_cpu_stack():
        torch.manual_seed(0)
        env = _env("base_quadrotor_with_gimbal_camera_imu", n=8)
        imu = env.imu
        env.imu.link_quat = torch.tensor([0.0, 0.0, np.sin(0.3), np.cos(0.3)], dtype=torch.float32)  # a rotated link
        for draw in (lambda: imu.reset(), lambda: env.reset_idx(torch.tensor([1, 4]))):
            draw()
            assert torch.equal(imu.mount_quats, quat_mul(imu.link_quat.expand_as(imu.sensor_quats), imu.sensor_quats))


def test_argument_validation():
    from aerial_gym_simulator_b200.config import robot_config as rc
    _register("_test_morphy_imu_nolink", rc.MorphyCompliantCfg, None)
    _register("_test_morphy_imu_badlink", rc.MorphyCompliantCfg, "no_such_link")
    _register("_test_morphy_imu_massless", rc.MorphyCompliantCfg, "connecting_link_0")
    with imu_cpu_stack():
        with pytest.raises(ValueError, match="joint reaction forces.*name the link with imu_config.parent_link"):
            _env("_test_morphy_imu_nolink")
        with pytest.raises(ValueError, match=r"no_such_link.*base_link"):
            _env("_test_morphy_imu_badlink")
        with pytest.raises(ValueError, match="connecting_link_0"):
            _env("_test_morphy_imu_massless")
        env = _env("morphy_compliant_imu", n=2)
        assert env.engine.imu_body == 0 and env.engine.imu_input.shape == (2, 9)
    # the C ABI: imu_body out of range, NULL output (checked before any launch)
    spec = H.spec_for("quad_attitude")
    _, art = morphy_compliant()
    from aerial_gym_simulator_b200.hp1 import build_config
    cfg = build_config(spec, 0)
    buf, s = _lib.AgxHp1Buffers(), art.to_struct()
    lib = _lib.load()
    out = torch.zeros(1, 9)
    for b, ptr, code in ((9, out.data_ptr(), -2), (-1, out.data_ptr(), -2), (0, None, -1), (8, out.data_ptr(), 0)):
        rc_ = lib.agx_hp1_articulated_step_imu(C.byref(cfg), C.byref(buf), C.byref(s), b, ptr, None)
        assert (rc_ == 0) == (code == 0), (b, rc_)
        if code:
            assert rc_ != 0 and (b"imu_body" in lib.agx_last_error() or b"imu_input" in lib.agx_last_error())
    with pytest.raises(ValueError, match="articulated"):
        from aerial_gym_simulator_b200.hp1 import Hp1Engine
        Hp1Engine._init_imu(type("E", (), {"articulation": None})(), 0)


# ---- machine code ----------------------------------------------------------------------------------------------------------------
# -Xptxas -v of the four instantiations of articulated_step_imu_kernel (CUDA 12.9, sm_90a): registers per thread.  The stack frame is
# the per-body arrays of the ABA, in local memory by design (articulated.cu), the same size as articulated_step_kernel's.
IMU_KERNEL_REGS = {(4, 9): 158, (4, 16): 158, (8, 9): 166, (8, 16): 166}
# normalised SASS (tools/sass_hash.py's idea, per function: comment lines and addresses dropped, encodings kept, the anonymous
# namespace's per-file hash masked) of every kernel articulated.cu had before the IMU entry point, md5
PARENT_SASS = {
    "articulated_body_state_kernelILi16E": "49fabc56648bbeedb676825c9dfce8b7",
    "articulated_body_state_kernelILi9E": "d6ab5ca7ca0215f6f63b3496123fa2d8",
    "articulated_step_kernelILi8ELi16E": "4d833f5c266d542fe19e29d2b82ef233",
    "articulated_step_kernelILi8ELi9E": "c2086c00bb11078baa2a0b9cc19015ce",
    "articulated_step_kernelILi4ELi16E": "61f12510a9b31d109fae04dc1a814d87",
    "articulated_step_kernelILi4ELi9E": "efbd4a3c22e2ad0447001440b6c8ac27",
}


@pytest.fixture(scope="module")
def articulated_unit():
    src = os.path.join(_build.CSRC, "articulated.cu")
    with tempfile.TemporaryDirectory() as d:
        obj = os.path.join(d, "articulated.o")
        r = subprocess.run([_build._nvcc()] + _build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o", obj], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        sass = subprocess.run([_build.cuda_tool("cuobjdump"), "-sass", obj], capture_output=True, text=True, check=True).stdout
    return r.stderr, sass


def sass_functions(txt):
    out, cur = {}, None
    for line in txt.splitlines():
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            cur = re.sub(r"_GLOBAL__N__\w+?_cu_\w{8}", "ANON", m.group(1))
            out[cur] = []
            continue
        s = line.strip()
        if cur is None or not s or s.startswith(("//", "...", ".")):
            continue
        out[cur].append(re.sub(r"/\*[0-9a-f]{4,}\*/", "", s))
    return {k: hashlib.md5("\n".join(v).encode()).hexdigest() for k, v in out.items()}


def test_imu_kernels_have_no_spills(articulated_unit):
    log, _ = articulated_unit
    blocks = re.findall(r"Compiling entry function '(\S+)'.*?\n(.*?spill loads)\n.*?Used (\d+) registers", log, re.S)
    found = {}
    for f, info, regs in blocks:
        m = re.search(r"articulated_step_imu_kernelILi(\d)ELi(\d+)E", f)
        if m:
            assert "0 bytes spill stores, 0 bytes spill loads" in info, (f, info)
            found[(int(m.group(1)), int(m.group(2)))] = int(regs)
    assert found == IMU_KERNEL_REGS, found


def test_pre_existing_kernels_keep_their_sass(articulated_unit):
    _, sass = articulated_unit
    h = sass_functions(sass)
    for key, md5 in PARENT_SASS.items():
        hits = [v for k, v in h.items() if key in k and "imu" not in k]
        assert hits == [md5], (key, hits)
