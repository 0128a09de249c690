"""Torque-driven (effort-mode) joints of articulated robots on the CPU (DESIGN.md "Articulated robots", "Torque-driven joints"): the
step of art_env_step<M, NB, IMU, true> (host shadow, tests/csrc/articulated_effort_shadow.cu) against oracle/articulated_effort_oracle.py,
the oracle itself against articulated_oracle, momentum conservation, an analytic two-body case and its clamp, and the host layer
(URDF, ArticulationSpec, Hp1Engine, EnvManager) on the CPU stack."""
import ctypes as C
import dataclasses
import os

import numpy as np
import pytest
import torch

from aerial_gym_simulator_b200 import _lib, urdf
from aerial_gym_simulator_b200.hp1 import ArticulationSpec, build_config
from oracle import articulated_effort_oracle as EO
from oracle import articulated_imu_oracle as IO
from oracle import articulated_oracle as AO

from . import _hp1_common as H
from ._cpu_stack_articulated import CpuArticulatedHp1Engine
from ._cpu_stack_articulated_effort import CpuEffortHp1Engine, effort_cpu_stack
from .test_articulated_cpu import (_urdf, check_substep, load_inputs, morphy_compliant, oracle_state, random_art, random_root, shaped_art,
                                   substep_inputs, table_of)
from .test_articulated_imu_cpu import _limit_crossing, gimbal_quad, sass_functions

RES = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "aerial_gym_simulator_b200", "resources", "robots")


def with_modes(art, modes, limit=None):
    """the ArticulationSpec `art` with drive_mode `modes` (and effort_limit `limit`, default the URDF's)"""
    return dataclasses.replace(art, drive_mode=modes, effort_limit=limit)


def effort_inputs(art, N, seed, over=1.5):
    """commands [N,D] float32: within +-over x the limit of a limited effort DOF (beyond it for |e| > limit), +-0.05 N m otherwise"""
    rng = np.random.default_rng(seed)
    E = np.where(art.effort_limit > 0, art.effort_limit * over, 0.05)
    return torch.tensor(rng.uniform(-1.0, 1.0, (N, art.num_dofs)) * E, dtype=torch.float32)


def run_effort(spec, art, inp, effort, physics_steps=1, imu_body=None):
    n = inp["root"].shape[0]
    eng = CpuEffortHp1Engine(spec, n, per_env_params="all", articulation=art, imu_body=imu_body)
    load_inputs(eng, inp)
    if eng.dof_actuation_force is not None:  # None without an effort DOF (a one-body tree)
        eng.dof_actuation_force.copy_(effort)
    eng.physics_step(inp["actions"], disturbance=inp["dist"], physics_steps=physics_steps)
    return eng


def reference_effort_substep(eng, spec, art, inp, effort, idx):
    model, st = oracle_state(eng, spec, inp, idx)
    ok = H.well_conditioned(model, st, inp["actions"][idx].double()).numpy()
    dof = inp["dof"][idx].double().numpy()
    ref = EO.substep(model, table_of(eng.art), st, dof[..., 0], dof[..., 1], inp["qs"][idx].double().numpy(),
                     inp["qds"][idx].double().numpy(), inp["actions"][idx].double(), art.effort_dof,
                     effort[idx].double().numpy(), np.float32(art.effort_limit).astype(np.float64), inp["dist"][idx].double())
    return ref, ok


# ---- the oracle itself -------------------------------------------------------------------------------------------------------
def _case(rng, B, M=4):
    art = random_art(rng, B, M=M)
    D = B - 1
    return art, table_of(art.to_struct()), random_root(rng), rng.uniform(-1, 1, D), rng.uniform(-2, 2, D), rng.uniform(-1, 1, D), \
        rng.uniform(-1, 1, D), rng.uniform(0, 2, M), rng.uniform(-1, 1, 3), rng.uniform(-0.05, 0.05, 3)


def test_oracle_without_torque_is_the_articulated_oracle():
    """no effort DOF: bit for bit articulated_oracle.dynamics; effort DOFs (k = 0) with zero command: the same as position DOFs
    with k = 0 and a zero velocity target"""
    rng = np.random.default_rng(1)
    grav, dt = np.array([0.0, 0.0, -9.81]), 0.01
    for _ in range(40):
        B = int(rng.integers(1, 17))
        art, tab, root, q, qd, qs, qds, th, F, T = _case(rng, B)
        D = B - 1
        ref = AO.dynamics(tab, root, q, qd, qs, qds, dt, grav, th, F, T)
        got = EO.dynamics(tab, root, q, qd, qs, qds, dt, grav, th, F, T, np.zeros(D, bool), rng.uniform(-1, 1, D), np.zeros(D))
        assert all(np.array_equal(a, b) for a, b in zip(ref, got))
        eff = rng.uniform(size=D) < 0.5
        tab["stiffness"][1:B][eff] = 0.0
        qds0 = np.where(eff, 0.0, qds)
        ref = AO.dynamics(tab, root, q, qd, qs, qds0, dt, grav, th, F, T)
        got = EO.dynamics(tab, root, q, qd, qs, qds, dt, grav, th, F, T, eff, np.zeros(D), rng.uniform(0, 1, D))
        assert all(np.array_equal(a, b) for a, b in zip(ref, got))


def test_oracle_internal_torque_conserves_momentum():
    """zero gravity, no thrust, no external force, the system at rest, dt -> 0 (H = M): the rate of the total spatial momentum
    sum_i I_i A_i is zero for any joint torques, on random trees"""
    rng = np.random.default_rng(2)
    for _ in range(40):
        B = int(rng.integers(2, 17))
        art, tab, root, q, _, qs, qds, _, _, _ = _case(rng, B)
        D = B - 1
        tab["stiffness"][:], tab["damping"][:] = 0.0, 0.0
        root[7:13] = 0.0
        z = np.zeros(D)
        e = rng.uniform(-0.1, 0.1, D)
        a0, qdd = EO.dynamics(tab, root, q, z, qs, qds, 0.0, np.zeros(3), np.zeros(4), np.zeros(3), np.zeros(3), np.ones(D, bool), e, z)
        assert np.abs(qdd).max() > 1.0  # the torques do move the tree
        R, P, V, A = IO.body_motion(tab, root, q, z, a0, qdd)
        hdot = np.zeros(6)
        for i in range(B):
            c = P[i] + R[i] @ tab["com"][i]
            hdot += AO.body_inertia(float(tab["mass"][i]), c, R[i] @ tab["inertia"][i] @ R[i].T) @ A[i]
        scale = sum(float(tab["mass"][i]) for i in range(B)) * np.abs(A).max()
        assert np.abs(hdot).max() <= 1e-12 * scale, hdot


def _two_body_table(J0=2e-3, J1=5e-4, m0=1.0, m1=0.2):
    """a base and one child on a z-axis joint 0.1 m above it, both COMs on that axis: z is principal for both"""
    z2 = np.zeros(2)
    return {"num_bodies": 2, "parent": np.array([-1, 0]), "joint_R": np.array([np.eye(3)] * 2), "joint_p": np.array([[0, 0, 0], [0, 0, 0.1]]),
            "axis": np.array([[0, 0, 0], [0, 0, 1.0]]), "mass": np.array([m0, m1]), "com": np.zeros((2, 3)),
            "inertia": np.array([np.diag([3e-3, 3e-3, J0]), np.diag([1e-3, 1e-3, J1])]), "stiffness": z2.copy(), "damping": z2.copy(),
            "motor_body": np.zeros(4, int), "motor_R": np.array([np.eye(3)] * 4), "motor_p": np.zeros((4, 3)), "motor_torque": np.zeros(4),
            "lower": z2, "upper": z2, "limited": np.zeros(2, int)}


def test_oracle_two_body_analytic_and_angular_momentum():
    """a constant torque tau on the joint of a free two-body tree in zero gravity: the base turns at -tau / J0, the joint at
    tau (1 / J0 + 1 / J1); integrated for 1 s (1,000 sub-steps), the angular momentum about the COM stays zero"""
    J0, J1, tau = 2e-3, 5e-4, 0.01
    tab = _two_body_table(J0, J1)
    root = np.zeros(13)
    root[6] = 1.0
    z3 = np.zeros(3)
    a0, qdd = EO.dynamics(tab, root, [0.3], [0.0], [0.0], [0.0], 0.0, z3, np.zeros(4), z3, z3, [True], [tau], [0.0])
    np.testing.assert_allclose(a0, [0, 0, -tau / J0, 0, 0, 0], atol=1e-12)
    np.testing.assert_allclose(qdd, [tau * (1 / J0 + 1 / J1)], rtol=1e-12)

    class Model:
        dt, linear_damping, angular_damping, max_linear_velocity, max_angular_velocity = 1e-3, 0.0, 0.0, 1e9, 1e9
    q, qd = np.array([0.3]), np.array([0.0])
    for _ in range(1000):
        a0, qdd = EO.dynamics(tab, root, q, qd, q, qd, Model.dt, z3, np.zeros(4), z3, z3, [True], [tau], [0.0])
        root, q, qd, _ = AO.integrate(Model, tab, root, a0, q, qd, qdd)
    lin, L = AO.momentum(tab, root, q, qd)
    assert np.abs(qd[0] - tau * (1 / J0 + 1 / J1)) < 1e-9 and np.abs(L).max() < 1e-12 and np.abs(lin).max() < 1e-12, (qd, L, lin)


def test_oracle_clamp_is_exact():
    E = np.array([0.1, 0.1, 0.1, 0.1, 0.0, 0.0])
    e = np.array([1.0, -1.0, 0.05, 0.1, 7.0, -7.0])
    assert np.array_equal(EO.effort_torque(e, E), [0.1, -0.1, 0.05, 0.1, 7.0, -7.0])
    assert EO.effort_torque(10 * 0.1, 0.1) == 0.1 and EO.effort_torque(-10 * 0.1, 0.1) == -0.1


# ---- the shadow against the oracle ------------------------------------------------------------------------------------------
def _check(spec, art, N, seed, cross=False, over=1.5):
    inp = substep_inputs(spec, art, N, seed)
    if cross:
        inp = _limit_crossing(inp, art)
    effort = effort_inputs(art, N, seed + 1, over)
    eng = run_effort(spec, art, inp, effort)
    idx = np.arange(N)
    ref, ok = reference_effort_substep(eng, spec, art, inp, effort, idx)
    assert ok.mean() > 0.8
    check_substep(eng, spec, inp, ref, ok, idx)
    return eng


@pytest.mark.parametrize("robot", ["morphy_compliant", "gimbal"])
def test_shadow_matches_oracle_on_shipped_robots(robot):
    """every DOF in effort mode, then alternate DOFs; commands inside and beyond the URDF limits; joints inside and crossing theirs"""
    spec = H.spec_for("quad_attitude")
    _, art = morphy_compliant() if robot == "morphy_compliant" else gimbal_quad()
    D = art.num_dofs
    for k, modes in enumerate(("effort", ["effort" if j % 2 == 0 else "position" for j in range(D)])):
        a = with_modes(art, modes)
        if robot == "morphy_compliant":
            a.damping[:] = np.where(a.effort_dof, 0.0, a.damping)
        if a.effort_dof.all() and not (a.bodies.urdf_damping[1:] > 0).all() and robot == "morphy_compliant":
            continue  # morphy's massless connecting links need a drive or URDF damping on their sweep joint
        for cross in (False, True):
            _check(spec, a, 24, 40 + 2 * k + cross, cross=cross)


def _effort_random_art(rng, B, M):
    art = shaped_art(rng, B, M=M, drive=True)
    D = B - 1
    modes = ["effort" if u < 0.5 else "position" for u in rng.uniform(size=D)]
    if D:
        modes[int(rng.integers(0, D))] = "effort"
    limit = np.where(rng.uniform(size=D) < 0.7, rng.uniform(0.01, 0.05, D), 0.0)
    return with_modes(art, modes, limit)


@pytest.mark.parametrize("M", [4, 8])
def test_shadow_matches_oracle_on_random_trees(M):
    rng = np.random.default_rng(80 + M)
    spec = H.spec_for("quad_attitude" if M == 4 else "octa_velocity")
    for B in range(1, 17):
        art = _effort_random_art(rng, B, M)
        _check(spec, art, 16, 600 + B, cross=bool(B % 3 == 0))


def test_zero_torque_is_bit_identical_to_the_plain_step_without_drive():
    """effort DOFs with zero command against the plain step with k = d = 0 (and zero velocity targets for the URDF damping)"""
    spec = H.spec_for("quad_attitude")
    rng = np.random.default_rng(5)
    for B in (2, 9, 16):
        art = shaped_art(rng, B, drive=True)
        art.bodies.urdf_damping[1:] = rng.uniform(0.0, 0.01, B - 1) * (rng.uniform(size=B - 1) < 0.5)
        eff = with_modes(art, "effort")
        plain_art = dataclasses.replace(art, stiffness=0.0, damping=0.0)
        inp = _limit_crossing(substep_inputs(spec, art, 32, 70 + B), art)
        inp["qds"].zero_()
        for steps in (0, 1, 3):
            plain = CpuArticulatedHp1Engine(spec, 32, per_env_params="all", articulation=plain_art)
            load_inputs(plain, inp)
            plain.physics_step(inp["actions"], disturbance=inp["dist"], physics_steps=steps)
            e = run_effort(spec, eff, inp, torch.zeros(32, B - 1), physics_steps=steps)
            for k in ("root_state", "motor_thrust", "dof_state") + CpuArticulatedHp1Engine.DERIVED:
                assert torch.equal(getattr(plain, k), getattr(e, k)), (B, steps, k)


def test_imu_variant_state_is_bit_identical():
    spec = H.spec_for("quad_attitude")
    _, art = gimbal_quad()
    art = with_modes(art, "effort")
    inp = _limit_crossing(substep_inputs(spec, art, 32, 12), art)
    effort = effort_inputs(art, 32, 13)
    for steps in (0, 1, 3):
        a = run_effort(spec, art, inp, effort, physics_steps=steps)
        b = run_effort(spec, art, inp, effort, physics_steps=steps, imu_body=art.bodies.num_bodies - 1)
        for k in ("root_state", "motor_thrust", "dof_state") + CpuArticulatedHp1Engine.DERIVED:
            assert torch.equal(getattr(a, k), getattr(b, k)), (steps, k)
        assert torch.isfinite(b.imu_input).all()


def test_clamp_ten_times_the_limit_is_the_limit():
    spec = H.spec_for("quad_attitude")
    _, art = gimbal_quad()
    art = with_modes(art, "effort")
    E = torch.tensor(art.effort_limit, dtype=torch.float32)
    assert (E == 0.1).all()
    inp = substep_inputs(spec, art, 16, 3)
    sign = torch.where(torch.arange(16)[:, None] % 2 == 0, 1.0, -1.0)
    a = run_effort(spec, art, inp, sign * E, physics_steps=3)
    b = run_effort(spec, art, inp, sign * 10 * E, physics_steps=3)
    for k in ("root_state", "dof_state"):
        assert torch.equal(getattr(a, k), getattr(b, k)), k
    c = run_effort(spec, art, inp, sign * 0.01 * E, physics_steps=3)  # (at E the stages reach their joint limits within the launch)
    assert not torch.equal(a.dof_state, c.dof_state)


# ---- host layer ----------------------------------------------------------------------------------------------------------------
def test_urdf_effort_limits():
    b = urdf.parse_urdf(os.path.join(RES, "quad", "quad_gimbal.urdf")).articulation()
    assert list(b.effort_limit) == [0.0, 0.1, 0.1]
    b = urdf.parse_urdf(os.path.join(RES, "morphy", "morphy_compliant.urdf")).articulation()
    assert list(b.effort_limit) == [0.0] + [1.0] * 8
    _, art = gimbal_quad()
    assert list(art.effort_limit) == [0.1, 0.1] and art.drive_mode == ["position", "position"] and not art.effort_dof.any()


def test_drive_mode_validation(tmp_path):
    _, art = gimbal_quad()
    for bad in ("torque", ["effort"], ["effort", "position", "effort"], ["effort", "velocity"]):
        with pytest.raises(ValueError, match="drive_mode"):
            with_modes(art, bad)
    with pytest.raises(ValueError, match="effort_limit"):
        with_modes(art, "effort", [-1.0, 0.1])
    a = with_modes(art, ["position", "effort"])
    assert a.stiffness[1] == 0.0 and a.damping[1] == 0.0 and a.stiffness[0] > 0  # the effort DOF's drive is off
    s = a.to_struct()
    assert s.stiffness[2] == 0.0 and s.damping[2] == np.float32(a.bodies.urdf_damping[2])
    # an effort DOF over a massless subtree without URDF damping has no pivot; with a drive gain it still has none
    b = _urdf(tmp_path, ["revolute"], mass=0.0).articulation()
    mk = lambda k, d, mode: ArticulationSpec(b, k, d, [0] * 4, np.tile(np.eye(3), (4, 1, 1)), np.zeros((4, 3)), np.zeros(4),
                                             drive_mode=mode)
    mk(1.0, 0.1, "position")
    with pytest.raises(ValueError, match="no inertia about the axis.*effort mode"):
        mk(1.0, 0.1, "effort")
    b.urdf_damping[1] = 0.01
    mk(0.0, 0.0, "effort")  # URDF damping makes the pivot non-zero


def test_urdf_negative_effort_raises(tmp_path):
    p = tmp_path / "n.urdf"
    p.write_text('<robot name="n"><link name="a"/><link name="b"><inertial><mass value="1"/>'
                 '<inertia ixx="1" iyy="1" izz="1" ixy="0" ixz="0" iyz="0"/></inertial></link>'
                 '<joint name="j" type="revolute"><parent link="a"/><child link="b"/><axis xyz="1 0 0"/>'
                 '<limit lower="-1" upper="1" effort="-2"/></joint></robot>')
    with pytest.raises(ValueError, match="negative <limit effort>"):
        urdf.parse_urdf(str(p)).articulation()


def test_c_abi_validation():
    lib = _lib.load()
    assert lib.agx_sizeof(17) == C.sizeof(_lib.AgxJointEffort) == 136
    spec = H.spec_for("quad_attitude")
    _, art = gimbal_quad()
    art = with_modes(art, "effort")
    buf, s, e = _lib.AgxHp1Buffers(), art.to_struct(), art.effort_struct()
    call = lambda n, eff, b=0, imu=None, st=s: lib.agx_hp1_articulated_step_effort(C.byref(build_config(spec, n)), C.byref(buf), C.byref(st),
                                                                                   eff, b, imu, None)
    out = torch.zeros(1, 9)
    assert call(0, C.byref(e)) == 0 and call(0, C.byref(e), 2, out.data_ptr()) == 0
    cases = [(lambda: call(0, None), b"effort is NULL"), (lambda: call(0, C.byref(e), 3, out.data_ptr()), b"imu_body"),
             (lambda: call(1, C.byref(e)), None)]
    for f, msg in cases[:2]:
        assert f() != 0 and msg in lib.agx_last_error()
    for bad in (-0.1, float("nan")):
        e2 = art.effort_struct()
        e2.effort_limit[1] = bad
        assert call(0, C.byref(e2)) != 0 and b"effort_limit[1]" in lib.agx_last_error()
    s2 = art.to_struct()
    s2.stiffness[2] = 0.5
    assert call(0, C.byref(e), st=s2) != 0 and b"stiffness[2]" in lib.agx_last_error()
    # one env with non-NULL state buffers and a NULL command array: rejected before any launch
    x = torch.zeros(64)
    buf.root_state, buf.motor_thrust, buf.actions = x.data_ptr(), x.data_ptr(), x.data_ptr()
    s.dof_state = s.dof_position_setpoint = s.dof_velocity_setpoint = x.data_ptr()
    assert call(1, C.byref(e)) != 0 and b"effort->effort is NULL" in lib.agx_last_error()


def _env(robot, env_name="empty_env", n=4, **args):
    from aerial_gym_simulator_b200.env_manager.env_manager import EnvManager
    return EnvManager("base_sim", env_name, robot, "lee_attitude_control", "cpu", num_envs=n, args={"seed": 1, **args})


def test_env_publishes_the_tensor_only_for_effort_robots():
    with effort_cpu_stack():
        torch.manual_seed(0)
        env = _env("base_quadrotor_with_torque_gimbal")
        gtd = env.global_tensor_dict
        t = gtd["dof_actuation_force_tensor"]
        assert t is env.engine.dof_actuation_force and t.shape == (4, 2) and (t == 0).all()
        assert list(env.engine.articulation.effort_limit) == [0.1, 0.1]
        env.reset()
        t.fill_(0.05)
        env.step(torch.zeros(4, 4))
        env.reset_idx(torch.tensor([0, 2]))
        env.reset()
        assert (t == 0.05).all()  # the user's: neither a step nor a reset writes it
        assert gtd["dof_actuation_force_tensor"].data_ptr() == t.data_ptr()
        for robot in ("base_quadrotor_with_gimbal_camera", "morphy_compliant"):
            env = _env(robot)
            assert "dof_actuation_force_tensor" not in env.global_tensor_dict and env.engine.dof_actuation_force is None


def test_torque_moves_the_gimbal_and_the_base_reacts():
    """a constant roll torque on the hovering quad: the roll stage spins up one way, the base the other"""
    with effort_cpu_stack():
        torch.manual_seed(0)
        env = _env("base_quadrotor_with_torque_gimbal", n=2)
        env.spec.enable_disturbance = False
        env.reset()
        gtd = env.global_tensor_dict
        st = gtd["robot_state_tensor"]
        st[:, 3:13] = 0.0
        st[:, 6] = 1.0
        gtd["dof_state_tensor"].zero_()
        gtd["dof_actuation_force_tensor"][:, 0] = torch.tensor([1e-4, -1e-4])
        env.step(torch.zeros(2, 4))
        qd = gtd["dof_state_tensor"][:, 0, 1]
        assert qd[0] > 0 and qd[1] < 0
        w = gtd["robot_angvel"]
        assert torch.sign(w[:, 0]).tolist() == [-1.0, 1.0]


# ---- machine code ----------------------------------------------------------------------------------------------------------------
# -Xptxas -v of the eight instantiations of articulated_step_effort_kernel<M, NB, IMU> (CUDA 12.9, sm_90a): registers per thread.  The
# stack frame is the per-body arrays of the ABA, in local memory by design (articulated.cu): 3,312 B at NB = 9, 5,856 B at NB = 16, the
# same as articulated_step_kernel's.  No spills.
EFFORT_KERNEL_REGS = {(4, 9, 0): 158, (4, 16, 0): 158, (8, 9, 0): 167, (8, 16, 0): 167,
                      (4, 9, 1): 158, (4, 16, 1): 158, (8, 9, 1): 167, (8, 16, 1): 167}
EFFORT_KERNEL_STACK = {9: 3312, 16: 5856}
# normalised SASS (test_articulated_imu_cpu.sass_functions), md5, of every step kernel articulated.cu had before the effort entry point
PARENT_SASS = {
    "articulated_step_kernelILi4ELi16E": "61f12510a9b31d109fae04dc1a814d87",
    "articulated_step_kernelILi4ELi9E": "efbd4a3c22e2ad0447001440b6c8ac27",
    "articulated_step_kernelILi8ELi16E": "4d833f5c266d542fe19e29d2b82ef233",
    "articulated_step_kernelILi8ELi9E": "c2086c00bb11078baa2a0b9cc19015ce",
    "articulated_step_imu_kernelILi4ELi16E": "126c2d9df2119902e827c3866d83e9fb",
    "articulated_step_imu_kernelILi4ELi9E": "2b321c922eed32aa91bc91d3594f5433",
    "articulated_step_imu_kernelILi8ELi16E": "f4eb229df3dcb4a243ca0d7daecea392",
    "articulated_step_imu_kernelILi8ELi9E": "8418465ed540f9c3753c25a8ffefbfff",
    "articulated_body_state_kernelILi16E": "49fabc56648bbeedb676825c9dfce8b7",
    "articulated_body_state_kernelILi9E": "d6ab5ca7ca0215f6f63b3496123fa2d8",
}


@pytest.fixture(scope="module")
def articulated_unit():
    import subprocess
    import tempfile

    from aerial_gym_simulator_b200 import _build
    src = os.path.join(_build.CSRC, "articulated.cu")
    with tempfile.TemporaryDirectory() as d:
        obj = os.path.join(d, "articulated.o")
        r = subprocess.run([_build._nvcc()] + _build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o", obj], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        sass = subprocess.run([_build.cuda_tool("cuobjdump"), "-sass", obj], capture_output=True, text=True, check=True).stdout
    return r.stderr, sass


def test_effort_kernels_have_no_spills(articulated_unit):
    import re
    log, _ = articulated_unit
    blocks = re.findall(r"Compiling entry function '(\S+)'.*?\n.*?(\d+) bytes stack frame, (.*?spill loads)\n.*?Used (\d+) registers", log,
                        re.S)
    found = {}
    for f, stack, info, regs in blocks:
        m = re.search(r"articulated_step_effort_kernelILi(\d)ELi(\d+)ELb(\d)E", f)
        if m:
            assert info == "0 bytes spill stores, 0 bytes spill loads", (f, info)
            assert int(stack) == EFFORT_KERNEL_STACK[int(m.group(2))], (f, stack)
            found[(int(m.group(1)), int(m.group(2)), int(m.group(3)))] = int(regs)
    assert found == EFFORT_KERNEL_REGS, found


def test_pre_existing_kernels_keep_their_sass(articulated_unit):
    _, sass = articulated_unit
    h = sass_functions(sass)
    for key, md5 in PARENT_SASS.items():
        hits = [v for k, v in h.items() if key in k and "effort" not in k]
        assert hits == [md5], (key, hits)
