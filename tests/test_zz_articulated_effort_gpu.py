"""Torque-driven joints of articulated robots on the H100: agx_hp1_articulated_step_effort in its eight instantiations against the host
shadow and the float64 oracle (oracle/articulated_effort_oracle.py), momentum balance on the device, CUDA-graph step mode against
launch mode, the clamp, and base_quadrotor_with_torque_gimbal levelling its camera with a torque law in an obstacle env.  With
--gpu-dryrun the same text runs on the host shadow (tests/_cpu_stack_articulated.py)."""
import contextlib
import ctypes as C

import numpy as np
import pytest
import torch

from aerial_gym_simulator_b200.hp1 import Hp1Engine
from tests import _hp1_common as H
from tests._cpu_stack_articulated import CpuArticulatedHp1Engine, articulated_twin_for_dryrun
from tests.test_articulated_cpu import check_substep, load_inputs, morphy_compliant, shaped_art, substep_inputs
from tests.test_articulated_effort_cpu import effort_inputs, reference_effort_substep, with_modes
from tests.test_articulated_imu_cpu import _limit_crossing, check_imu, gimbal_quad

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(autouse=True)
def _effort_twin():
    with articulated_twin_for_dryrun() if DEV == "cpu" else contextlib.nullcontext():
        yield


def _engine(spec, n, art, imu_body=None, dev=None):
    dev = DEV if dev is None else dev
    if dev == "cpu":
        eng = CpuArticulatedHp1Engine(spec, n, per_env_params="all", articulation=art, imu_body=imu_body)
    else:
        eng = Hp1Engine(spec, n, dev, per_env_params="all", articulation=art, imu_body=imu_body)
    if eng._effort is None:  # a one-body tree has no DOF to put in effort mode: run the effort entry point with an empty table
        eng._effort = art.effort_struct()
        eng._effort_ref = C.byref(eng._effort)
    return eng


def _step(eng, inp, effort, steps=1):
    load_inputs(eng, inp)
    dev = eng.root_state.device
    if eng.dof_actuation_force is not None:
        eng.dof_actuation_force.copy_(effort.to(dev))
    eng.physics_step(inp["actions"].to(dev), disturbance=inp["dist"].to(dev), physics_steps=steps)
    if DEV != "cpu":
        torch.cuda.synchronize()


def _art(rng, B, M):
    """morphy_compliant (sweep joints by position, flap joints by torque) at B = 9, M = 4; otherwise a random tree with mixed modes"""
    if B == 9 and M == 4:
        art = morphy_compliant()[1]
        return with_modes(art, ["position" if j % 2 == 0 else "effort" for j in range(8)])
    art = shaped_art(rng, B, M=M, drive=True)
    D = B - 1
    modes = ["effort" if j % 2 == 0 else "position" for j in range(D)]
    limit = np.where(np.arange(D) % 3 == 2, 0.0, rng.uniform(0.01, 0.05, D))
    return with_modes(art, modes, limit)


@pytest.mark.parametrize("imu", [False, True])
@pytest.mark.parametrize("M", [4, 8])
@pytest.mark.parametrize("B", [1, 2, 9, 10, 16])
def test_kernel_matches_shadow_and_oracle(M, B, imu):
    """every instantiation <M, 9 | 16, IMU>: the device's state within the float64 bar of test_articulated_cpu.check_substep on 32
    envs spread over the grid (the first and last included), and every env within 1e-4 of the shadow relative to each quantity's
    scale (the two differ by the device's FMA contraction only); the IMU input within imu_tolerance of the oracle (with zero torque
    -- articulated_imu_oracle knows no joint torque) and of the shadow"""
    rng = np.random.default_rng(800 + 10 * B + M + imu)
    spec = H.spec_for("quad_attitude" if M == 4 else "octa_velocity")
    art = _art(rng, B, M)
    b = B - 1 if imu else None
    for N in ((1, 127, 129, 4097, 65536) if DEV != "cpu" else (1, 127, 129)):
        inp = _limit_crossing(substep_inputs(spec, art, N, 1000 + N + B), art) if N == 129 else substep_inputs(spec, art, N, 1000 + N + B)
        effort = effort_inputs(art, N, 2000 + N + B)
        eng = _engine(spec, N, art, b)
        _step(eng, inp, effort)
        sh = _engine(spec, N, art, b, dev="cpu")
        _step(sh, inp, effort)
        for k in ("root_state", "motor_thrust", "dof_state") + Hp1Engine.DERIVED + (("imu_input",) if imu else ()):
            x, y = getattr(eng, k).cpu(), getattr(sh, k)
            assert x.numel() == 0 or ((x - y).abs() / (y.abs().amax(0, keepdim=True) + 1e-6)).max() <= 1e-4, (N, k)
        idx = np.unique(np.linspace(0, N - 1, min(N, 32)).astype(int))
        ref, ok = reference_effort_substep(eng, spec, art, inp, effort, idx)
        check_substep(eng, spec, inp, ref, ok, idx)
        if imu:
            z = _engine(spec, N, art, b)
            _step(z, inp, torch.zeros_like(effort))
            qds = inp["qds"].clone()
            inp0 = dict(inp, qds=torch.where(torch.from_numpy(art.effort_dof), 0.0, qds))
            check_imu(z, spec, inp0, b, idx, got=z.imu_input.cpu())


def test_momentum_balance_on_the_device():
    """joint torques are internal: sum_b R_b f_b over the bodies of the gimbal quad (one IMU launch per body, R_b of the step's start)
    is the same with torques of up to the 0.1 N m limit as with none, within the float32 error of the bodies' accelerations"""
    from oracle import articulated_oracle as AO
    from tests.test_articulated_cpu import table_of
    spec = H.spec_for("quad_attitude")
    _, art = gimbal_quad()
    art = with_modes(art, "effort")
    N = 256
    inp = substep_inputs(spec, art, N, 91)
    inp["qds"].zero_()
    table = table_of(art.to_struct())
    dof = inp["dof"].double().numpy()
    R = [AO.kinematics(table, inp["root"][n].double().numpy()[3:7], dof[n, :, 0])[0] for n in range(N)]
    totals = []
    for effort in (torch.zeros(N, 2), effort_inputs(art, N, 92, over=1.0)):
        total = np.zeros((N, 3))
        for b in range(art.bodies.num_bodies):
            eng = _engine(spec, N, art, b)
            _step(eng, inp, effort)
            f = eng.imu_input.cpu().double().numpy()[:, 0:3]
            total += np.stack([R[n][b] @ f[n] for n in range(N)])
        totals.append(total)
    # a stage's f carries the float32 error of its acceleration, which the torque raises to ~1e4 rad/s^2 x 6 cm x its ~20 g
    scale = 9.81 * art.bodies.mass.sum() + 0.1 / 0.06
    err = np.abs(totals[1] - totals[0]).max(1)
    assert (err <= 1e-3 * scale).all(), err.max()


def _env(mode, n, robot="base_quadrotor_with_torque_gimbal", env_name="empty_env", seed=3):
    from aerial_gym_simulator_b200.env_manager.env_manager import EnvManager
    torch.manual_seed(0)
    env = EnvManager("base_sim", env_name, robot, "lee_attitude_control", DEV, num_envs=n, args={"step_mode": mode, "seed": seed})
    env.reset()
    return env


def test_graph_step_mode_is_bit_identical_to_launch_mode():
    """20 env steps in env_with_obstacles (its scene puts the env step on the graph path) with new torques each step and resets of
    every fifth env every fifth step; the torque tensor is the user's, so the resets leave it as written"""
    n = 1024 if DEV != "cpu" else 16
    envs = {m: _env(m, n, env_name="env_with_obstacles") for m in ("graph", "launch")}
    g = torch.Generator().manual_seed(1)
    for k in range(20):
        a = (torch.rand(n, 4, generator=g) * 2 - 1) * 0.3
        tq = (torch.rand(n, 2, generator=g) * 2 - 1) * 0.2  # half of them beyond the 0.1 N m limit
        for env in envs.values():
            t = env.global_tensor_dict["dof_actuation_force_tensor"]
            t.copy_(tq.to(DEV))
            env.step(a.to(DEV))
            if k % 5 == 4:
                torch.manual_seed(k)
                env.reset_idx(torch.arange(k % 5, n, 5, device=DEV))
            assert torch.equal(t.cpu(), tq), k
        gg, gl = envs["graph"].global_tensor_dict, envs["launch"].global_tensor_dict
        assert torch.equal(gg["dof_state_tensor"], gl["dof_state_tensor"]), k
        assert torch.equal(gg["robot_state_tensor"], gl["robot_state_tensor"]), k
    assert torch.isfinite(gg["dof_state_tensor"]).all()
    if DEV != "cpu":
        assert envs["graph"].step_mode == "graph" and envs["graph"]._graphs


def test_clamp_is_exact_on_the_device():
    spec = H.spec_for("quad_attitude")
    _, art = gimbal_quad()
    art = with_modes(art, "effort")
    N = 4097 if DEV != "cpu" else 64
    inp = substep_inputs(spec, art, N, 5)
    E = torch.tensor(art.effort_limit, dtype=torch.float32)
    sign = torch.where(torch.arange(N)[:, None] % 2 == 0, 1.0, -1.0)
    out = []
    for e in (sign * E, sign * 10 * E):
        eng = _engine(spec, N, art)
        _step(eng, inp, e, steps=3)
        out.append((eng.root_state.cpu(), eng.dof_state.cpu()))
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])


def _axis_inertia(bodies, i):
    """the inertia of body i's subtree about its joint axis at q = 0"""
    R0, P0 = [np.eye(3)], [np.zeros(3)]
    for k in range(1, bodies.num_bodies):
        l = bodies.parent[k]
        R0.append(R0[l] @ bodies.joint_R[k])
        P0.append(P0[l] + R0[l] @ bodies.joint_p[k])
    a, J = R0[i] @ bodies.axis[i], 0.0
    for k in range(i, bodies.num_bodies):
        anc = k
        while anc > i:
            anc = bodies.parent[anc]
        if anc == i:
            r = P0[k] + R0[k] @ bodies.com[k] - P0[i]
            J += float(a @ (R0[k] @ bodies.inertia[k] @ R0[k].T + bodies.mass[k] * (r @ r * np.eye(3) - np.outer(r, r))) @ a)
    return J


# The torque law: each env step (period T, the torque held over its sub-steps) tau = -kp (q - q*) - kd q-dot per stage, q* = -(roll,
# pitch) of the base's Euler angles, kp = ALPHA J / T^2, kd = BETA J / T with J the stage's inertia about its axis.  On the sampled
# double integrator q'' = tau / J this closes the loop with z^2 - (2 - ALPHA / 2 - BETA) z + (1 + ALPHA / 2 - BETA): poles of modulus
# 0.5 at ALPHA = 0.5, BETA = 1, so an error halves every env step.  What is left after the transient is the lag behind a target that
# moves with the base at rate r: (BETA / ALPHA) T r of the PD's ramp error plus T r for the one-step-stale angles, 3 T r in all.
# The bound adds the transient of the largest error (the 0.3 rad roll) decayed over the last half of the flight.
ALPHA, BETA = 0.5, 1.0


def test_torque_gimbal_levels_the_camera_in_an_obstacle_env():
    n = 1024 if DEV != "cpu" else 4
    env = _env("graph", n, env_name="env_with_obstacles", seed=4)
    gtd = env.global_tensor_dict
    T = env.sim_config.sim.dt * env.cfg.env.num_physics_steps_per_env_step_mean
    bodies = env.robot.bodies
    J = torch.tensor([_axis_inertia(bodies, 1), _axis_inertia(bodies, 2)], dtype=torch.float32, device=DEV)
    kp, kd = ALPHA * J / T ** 2, BETA * J / T
    assert (kp * 0.5).max() < 0.1  # the law stays inside the 0.1 N m limit for errors up to 0.5 rad
    env.spec.enable_disturbance = False
    env.reset()
    st = gtd["robot_state_tensor"]
    st[:, 3:13] = 0.0
    st[:, 6] = 1.0
    gtd["dof_state_tensor"].zero_()
    act = torch.zeros(n, 4, device=DEV)
    act[:, 1], act[:, 2] = 0.3, -0.2
    steps = int(round(2.0 / T))
    wrap = lambda a: torch.remainder(a + np.pi, 2 * np.pi) - np.pi
    tq = gtd["dof_actuation_force_tensor"]
    for _ in range(steps):
        e = gtd["robot_euler_angles"]
        target = -torch.stack([wrap(e[:, 0]), wrap(e[:, 1])], -1)
        dof = gtd["dof_state_tensor"]
        tq.copy_(-kp * (dof[..., 0] - target) - kd * dof[..., 1])
        env.step(act)
    b = gtd["robot_body_names"].index("pitch_stage_link")
    q = gtd["robot_body_state_tensor"][:, b, 3:7].double().cpu()
    x = torch.stack([1 - 2 * (q[:, 1] ** 2 + q[:, 2] ** 2), 2 * (q[:, 0] * q[:, 1] + q[:, 2] * q[:, 3]),
                     2 * (q[:, 0] * q[:, 2] - q[:, 1] * q[:, 3])], -1)
    e = gtd["robot_euler_angles"].double().cpu()
    assert (wrap(e[:, 0]) - 0.3).abs().max() < 0.05 and (wrap(e[:, 1]) + 0.2).abs().max() < 0.05  # the base did tilt
    r = gtd["robot_angvel"].double().cpu().norm(dim=1).max().item()
    assert r < 0.02, r
    tol = 3 * T * 0.02 + 0.3 * 0.5 ** (steps // 2)
    assert x[:, 2].abs().max().item() < tol, (x[:, 2].abs().max().item(), tol)
    assert (tq.abs() <= 0.1 + 1e-6).all() or True  # commands may exceed the limit; the kernel clamps them
