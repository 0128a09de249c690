"""Joint force sensing of articulated robots on the H100: agx_hp1_articulated_step_joint_force in its four instantiations against the
host shadow and the float64 oracle (oracle/articulated_joint_force_oracle.py), the base's momentum balance on the device, the state
against the plain kernel, CUDA-graph step mode against launch mode, and the clamp.  With --gpu-dryrun the same text runs on the host
shadow (tests/_cpu_stack_articulated_joint_force.py)."""
import contextlib

import numpy as np
import pytest
import torch

from aerial_gym_simulator_b200.hp1 import Hp1Engine
from tests import _cpu_stack_articulated_joint_force as CJ
from tests import _hp1_common as H
from tests.test_articulated_cpu import load_inputs, morphy_compliant, shaped_art, substep_inputs
from tests.test_articulated_cpu import check_substep
from tests.test_articulated_effort_cpu import effort_inputs, reference_effort_substep, with_modes
from tests.test_articulated_imu_cpu import _limit_crossing, gimbal_quad
from tests.test_articulated_joint_force_cpu import check_joint_force

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
STATE = ("root_state", "motor_thrust", "dof_state") + Hp1Engine.DERIVED


@pytest.fixture(autouse=True)
def _jf_twin():
    with CJ.joint_force_twin_for_dryrun() if DEV == "cpu" else contextlib.nullcontext():
        yield


def _engine(spec, n, art, imu_body=None, dev=None, joint_force=True):
    dev = DEV if dev is None else dev
    if dev == "cpu":
        return CJ.CpuJointForceHp1Engine(spec, n, per_env_params="all", articulation=art, imu_body=imu_body, joint_force=joint_force)
    return Hp1Engine(spec, n, dev, per_env_params="all", articulation=art, imu_body=imu_body, joint_force=joint_force)


def _step(eng, inp, effort=None, steps=1):
    load_inputs(eng, inp)
    dev = eng.root_state.device
    if eng.dof_actuation_force is not None:
        eng.dof_actuation_force.copy_(effort.to(dev))
    eng.physics_step(inp["actions"].to(dev), disturbance=inp["dist"].to(dev), physics_steps=steps)
    if DEV != "cpu":
        torch.cuda.synchronize()


def _art(rng, B, M, effort):
    """morphy_compliant at B = 9, M = 4 (its flap joints by torque with `effort`); otherwise a random tree, alternate DOFs by torque"""
    if B == 9 and M == 4:
        art = morphy_compliant()[1]
        return with_modes(art, ["position" if j % 2 == 0 else "effort" for j in range(8)]) if effort else art
    art = shaped_art(rng, B, M=M, drive=True)
    if not effort or B == 1:
        return art
    D = B - 1
    limit = np.where(np.arange(D) % 3 == 2, 0.0, rng.uniform(0.01, 0.05, D))
    return with_modes(art, ["effort" if j % 2 == 0 else "position" for j in range(D)], limit)


@pytest.mark.parametrize("variant", ["plain", "imu", "effort", "imu+effort"])
@pytest.mark.parametrize("M", [4, 8])
@pytest.mark.parametrize("B", [1, 2, 9, 10, 16])
def test_kernel_matches_shadow_and_oracle(M, B, variant):
    """every instantiation <M, 9 | 16>, with and without the IMU input and effort DOFs, on 32 envs spread over the grid (the first and
    last included): joint_wrench and dof_force within jf_tolerance of the float64 oracle, dof_force against the drive law at the
    device's own end-of-step state (check_dof_force_identity, per joint), and the state within check_substep's float64 bar, per
    component.  Against the shadow, every env within 1e-3 of each quantity's largest magnitude over the grid: the two differ by the
    device's FMA contraction, which these trees' light bodies amplify through joint accelerations of 1e3-1e4 rad/s^2, and some
    columns (the rows of massless links) hold only rounding noise of ~1e-8 N, so a per-column relative bar would measure noise;
    the per-component checks are the float64 ones above."""
    rng = np.random.default_rng(1200 + 10 * B + M)
    spec = H.spec_for("quad_attitude" if M == 4 else "octa_velocity")
    art = _art(rng, B, M, "effort" in variant)
    b = B - 1 if "imu" in variant else None
    for N in ((1, 127, 129, 4097, 65536) if DEV != "cpu" else (1, 127, 129)):
        inp = substep_inputs(spec, art, N, 3000 + N + B)
        if N == 129:
            inp = _limit_crossing(inp, art)
        effort = effort_inputs(art, N, 4000 + N + B) if art.effort_dof.any() else None
        eng = _engine(spec, N, art, b)
        _step(eng, inp, effort)
        sh = _engine(spec, N, art, b, dev="cpu")
        _step(sh, inp, effort)
        keys = ("joint_wrench", "dof_force") + STATE + (("imu_input",) if b is not None else ())
        for k in keys:
            x, y = getattr(eng, k).cpu(), getattr(sh, k)
            r = 0.0 if x.numel() == 0 else float((x - y).abs().max() / (y.abs().max() + 1e-6))
            assert r <= 1e-3, (N, k, r)
        idx = np.unique(np.linspace(0, N - 1, min(N, 32)).astype(int))
        check_joint_force(eng, spec, inp, art, idx, effort)  # includes the dof_force identity on the device's own outputs
        ref, ok = reference_effort_substep(eng, spec, art, inp, effort if effort is not None else torch.zeros(N, B - 1), idx)
        check_substep(eng, spec, inp, ref, ok, idx)


def test_base_momentum_balance_on_the_device():
    """morphy_compliant at 4,096 envs: the base's Newton-Euler balance from the device's rows -- the thrusts, drag, disturbance and
    gravity on the base minus what its children's joints take, in world axes, equals the base's rate of momentum m_0 a_c,0 -- within
    the float32 error of the joint rows' forces"""
    from oracle import articulated_imu_oracle as IO
    from oracle import articulated_joint_force_oracle as JO
    from tests.test_articulated_cpu import oracle_state, table_of
    spec = H.spec_for("quad_attitude")
    _, art = morphy_compliant()
    N = 4096 if DEV != "cpu" else 64
    inp = substep_inputs(spec, art, N, 77)
    eng = _engine(spec, N, art, imu_body=0)
    _step(eng, inp)
    W = eng.joint_wrench.cpu().double().numpy()
    f0 = eng.imu_input.cpu().double().numpy()[:, 0:3]  # m_0 R_0^T (a_c,0 - g): the base's rate of momentum less gravity
    table = table_of(eng.art)
    idx = np.arange(N)
    model, st = oracle_state(eng, spec, inp, idx)
    ok = H.well_conditioned(model, st, inp["actions"].double()).numpy()
    thrust, F_w, _ = IO.substep_inputs(model, st, inp["actions"].double(), inp["dist"].double())
    dof = inp["dof"].double().numpy()
    children = [i for i in range(1, table["num_bodies"]) if table["parent"][i] == 0]
    worst = 0.0
    for n in np.flatnonzero(ok)[:: max(1, N // 512)]:
        R, P = JO.newton_euler(table, st.root[n].numpy(), dof[n, :, 0], dof[n, :, 1], np.zeros(6), np.zeros(8), model.gravity, thrust[n],
                               F_w[n], np.zeros(3))[1:]
        fext = JO.external_forces(table, R, P, np.zeros(3), thrust[n], F_w[n], np.zeros(3))[0, 3:]
        reac = sum(R[c] @ W[n, c, 0:3] for c in children)
        err = np.abs(R[0] @ f0[n] - (fext - reac)).max()
        scale = np.abs(thrust[n]).sum() + 9.81 * table["mass"].sum()
        worst = max(worst, err / scale)
    assert worst <= 1e-4, worst


def test_state_matches_the_plain_kernel():
    """a separate compilation: the state after 3 sub-steps equals the plain kernel's to float32 rounding"""
    spec = H.spec_for("quad_attitude")
    _, art = morphy_compliant()
    N = 4097 if DEV != "cpu" else 64
    inp = substep_inputs(spec, art, N, 5)
    a, p = _engine(spec, N, art), _engine(spec, N, art, joint_force=False)
    _step(a, inp, steps=3)
    _step(p, inp, steps=3)
    for k in STATE:
        x, y = getattr(a, k).cpu(), getattr(p, k).cpu()
        assert ((x - y).abs() / (y.abs().amax(0, keepdim=True) + 1e-6)).max() <= 1e-5, k


def _register(name, base):
    from aerial_gym_simulator_b200.registry._core import robot_registry
    from aerial_gym_simulator_b200.robots import ArticulatedMultirotor

    class Cfg(base):
        class joint_config(base.joint_config):
            enable_dof_force_sensors = True

        class sensor_config(base.sensor_config):
            enable_imu = True

            class imu_config(base.sensor_config.imu_config):
                parent_link = "gimbal_camera_link"
    robot_registry.register(name, ArticulatedMultirotor, Cfg)
    return name


def test_graph_step_mode_is_bit_identical_to_launch_mode():
    """20 env steps of the torque gimbal with an IMU on its camera link in env_with_obstacles (its scene puts the env step on the graph
    path), new torques each step and resets of every fifth env every fifth step"""
    from aerial_gym_simulator_b200.config import robot_config as rc
    from aerial_gym_simulator_b200.env_manager.env_manager import EnvManager
    name = _register("_test_torque_gimbal_jf_imu", rc.BaseQuadWithTorqueGimbalCfg)
    n = 1024 if DEV != "cpu" else 16
    envs = {}
    for mode in ("graph", "launch"):
        torch.manual_seed(0)
        envs[mode] = EnvManager("base_sim", "env_with_obstacles", name, "lee_attitude_control", DEV, num_envs=n,
                                args={"step_mode": mode, "seed": 3})
        envs[mode].reset()
    g = torch.Generator().manual_seed(1)
    for k in range(20):
        a = (torch.rand(n, 4, generator=g) * 2 - 1) * 0.3
        tq = (torch.rand(n, 2, generator=g) * 2 - 1) * 0.2
        for env in envs.values():
            env.global_tensor_dict["dof_actuation_force_tensor"].copy_(tq.to(DEV))
            env.step(a.to(DEV))
            if k % 5 == 4:
                torch.manual_seed(k)
                env.reset_idx(torch.arange(k % 5, n, 5, device=DEV))
        gg, gl = envs["graph"].global_tensor_dict, envs["launch"].global_tensor_dict
        for key in ("dof_force_tensor", "robot_joint_wrench_tensor", "dof_state_tensor", "robot_state_tensor"):
            assert torch.equal(gg[key], gl[key]), (k, key)
        assert torch.equal(envs["graph"].engine.imu_input, envs["launch"].engine.imu_input), k
    assert (gg["robot_joint_wrench_tensor"][:, 1:] != 0).any()
    if DEV != "cpu":
        assert envs["graph"].step_mode == "graph" and envs["graph"]._graphs


def test_ten_times_the_limit_gives_the_same_outputs():
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
        out.append([getattr(eng, k).cpu() for k in ("root_state", "dof_state", "joint_wrench", "dof_force")])
    assert all(torch.equal(x, y) for x, y in zip(*out))
