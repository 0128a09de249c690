"""The IMU on a link of an articulated robot on the H100: agx_hp1_articulated_step_imu in its four instantiations against the host
shadow and the float64 oracle (oracle/articulated_imu_oracle.py), its state outputs against agx_hp1_articulated_step's,
momentum balance over one launch per body, CUDA-graph step mode against launch mode with imu_measurement, and the gimbal IMU end to
end.  With --gpu-dryrun the same text runs on the host shadow (tests/_cpu_stack_articulated.py)."""
import contextlib

import numpy as np
import pytest
import torch

from aerial_gym_simulator_b200.hp1 import Hp1Engine
from tests import _hp1_common as H
from tests._cpu_stack_articulated import CpuArticulatedHp1Engine, articulated_twin_for_dryrun
from tests.test_articulated_cpu import check_substep, load_inputs, morphy_compliant, reference_substep, shaped_art, substep_inputs
from tests.test_articulated_imu_cpu import check_imu

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(autouse=True)
def _imu_twin():
    with articulated_twin_for_dryrun() if DEV == "cpu" else contextlib.nullcontext():
        yield


def _engine(spec, n, art, b):
    if DEV == "cpu":
        return CpuArticulatedHp1Engine(spec, n, per_env_params="all", articulation=art, imu_body=b)
    return Hp1Engine(spec, n, DEV, per_env_params="all", articulation=art, imu_body=b)


def _plain(spec, n, art):
    if DEV == "cpu":
        return CpuArticulatedHp1Engine(spec, n, per_env_params="all", articulation=art)
    return Hp1Engine(spec, n, DEV, per_env_params="all", articulation=art)


def _step(eng, inp, steps=1):
    load_inputs(eng, inp)
    eng.physics_step(inp["actions"].to(eng.root_state.device), disturbance=inp["dist"].to(eng.root_state.device), physics_steps=steps)
    if DEV != "cpu":
        torch.cuda.synchronize()


@pytest.mark.parametrize("M", [4, 8])
@pytest.mark.parametrize("B", [1, 2, 9, 10, 16])
def test_kernel_matches_shadow_and_oracle(M, B):
    """every instantiation <M, 9 | 16>: the device's imu_input within imu_tolerance of the oracle on 32 envs spread over the grid (the
    first and last included), every env within 1e-4 of the shadow relative to the IMU input's scale (the two differ by the device's
    FMA contraction only), and the state within float32 rounding of agx_hp1_articulated_step's"""
    rng = np.random.default_rng(700 + 10 * B + M)
    spec = H.spec_for("quad_attitude" if M == 4 else "octa_velocity")
    art = morphy_compliant()[1] if (B == 9 and M == 4) else shaped_art(rng, B, M=M, drive=bool(B % 2))
    b = B - 1
    for N in ((1, 127, 129, 4097, 65536) if DEV != "cpu" else (1, 127, 129)):
        inp = substep_inputs(spec, art, N, 900 + N + B)
        eng = _engine(spec, N, art, b)
        _step(eng, inp)
        plain = _plain(spec, N, art)
        _step(plain, inp)
        # the state: on the host shadow bit-identical to the plain step (test_articulated_imu_cpu.py); on the device the two kernels
        # are compiled separately and ptxas contracts multiply-adds differently, so here they agree to float32 rounding, and both
        # meet the float64 bar of test_articulated_cpu.check_substep
        for k in ("root_state", "motor_thrust", "dof_state") + Hp1Engine.DERIVED:
            x, y = getattr(eng, k).cpu(), getattr(plain, k).cpu()
            assert x.numel() == 0 or ((x - y).abs() / (y.abs().amax(0, keepdim=True) + 1e-6)).max() <= 1e-4, (N, k)
        idx = np.unique(np.linspace(0, N - 1, min(N, 32)).astype(int))
        ref, ok = reference_substep(eng, spec, art, inp, idx)
        check_substep(eng, spec, inp, ref, ok, idx)
        got = eng.imu_input.cpu()
        sh = CpuArticulatedHp1Engine(spec, N, per_env_params="all", articulation=art, imu_body=b)
        _step_cpu = (lambda e: (load_inputs(e, inp), e.physics_step(inp["actions"], disturbance=inp["dist"], physics_steps=1)))
        _step_cpu(sh)
        scale = sh.imu_input.abs().amax(0, keepdim=True) + 1e-6
        assert ((got - sh.imu_input).abs() / scale).max() <= 1e-4
        check_imu(eng, spec, inp, b, idx, got=got)


def test_momentum_balance_on_the_device():
    """one launch per imu_body from the same state: sum_b R_b f_b (R_b of the step's start, from the oracle's kinematics) = the world
    sum of the thrusts and the base's drag + disturbance, per env"""
    from oracle import articulated_imu_oracle as IO
    from oracle import articulated_oracle as AO
    from tests.test_articulated_cpu import oracle_state, table_of
    spec = H.spec_for("quad_attitude")
    _, art = morphy_compliant()
    N = 256
    inp = substep_inputs(spec, art, N, 77)
    total = np.zeros((N, 3))
    table = table_of(art.to_struct())
    dof = inp["dof"].double().numpy()
    for b in range(art.bodies.num_bodies):
        if not art.bodies.mass[b] > 0:
            continue
        eng = _engine(spec, N, art, b)
        _step(eng, inp)
        f = eng.imu_input.cpu().double().numpy()[:, 0:3]
        for n in range(N):
            R, _, _ = AO.kinematics(table, inp["root"][n].double().numpy()[3:7], dof[n, :, 0])
            total[n] += R[b] @ f[n]
    model, st = oracle_state(eng, spec, inp, np.arange(N))
    ok = H.well_conditioned(model, st, inp["actions"].double()).numpy()
    thrust, F_w, _ = IO.substep_inputs(model, st, inp["actions"].double(), inp["dist"].double())
    ext = F_w.copy()
    for n in range(N):
        R, _, _ = AO.kinematics(table, inp["root"][n].double().numpy()[3:7], dof[n, :, 0])
        for k in range(4):
            ext[n] += (R[int(table["motor_body"][k])] @ table["motor_R"][k])[:, 2] * thrust[n, k]
    # each body's f carries the float32 error of its acceleration (imu_tolerance's E_lin ~ 2e-4 amax per level); 1e-3 of the total
    # thrust and weight bounds their sum over the nine bodies
    scale = np.abs(thrust).sum(1) + 9.81 * art.bodies.mass.sum()
    err = np.abs(total - ext).max(1)
    assert (err[ok] <= 1e-3 * scale[ok]).all(), err.max()


def _env(mode, n, robot="morphy_compliant_imu"):
    from aerial_gym_simulator_b200.env_manager.env_manager import EnvManager
    torch.manual_seed(0)
    env = EnvManager("base_sim", "empty_env", robot, "lee_attitude_control", DEV, num_envs=n, args={"step_mode": mode, "seed": 3})
    env.reset()
    return env


def test_graph_step_mode_imu_is_bit_identical_to_launch_mode():
    """20 env steps with resets of every fifth env every fifth step, render() after each (morphy_compliant draws disturbances: the
    graph path); the IMU's torch draws are seeded alike for both managers"""
    n = 1024 if DEV != "cpu" else 64
    envs = {m: _env(m, n) for m in ("graph", "launch")}
    for env in envs.values():
        env.global_tensor_dict["dof_position_setpoint_tensor"].fill_(0.1)
    g = torch.Generator().manual_seed(1)
    for k in range(20):
        a = (torch.rand(n, 4, generator=g) * 2 - 1) * 0.3
        for env in envs.values():
            env.step(a.to(DEV))
            if k % 5 == 4:
                torch.manual_seed(k)
                env.reset_idx(torch.arange(k % 5, n, 5, device=DEV))
            torch.manual_seed(100 + k)
            env.render()
        gg, gl = envs["graph"].global_tensor_dict, envs["launch"].global_tensor_dict
        assert torch.equal(envs["graph"].engine.imu_input, envs["launch"].engine.imu_input), k
        assert torch.equal(gg["imu_measurement"], gl["imu_measurement"]), k
        assert torch.equal(gg["robot_state_tensor"], gl["robot_state_tensor"]), k
    assert torch.isfinite(gg["imu_measurement"]).all()
    if DEV != "cpu":
        assert envs["graph"].step_mode == "graph" and envs["graph"]._graphs


def test_gimbal_imu_end_to_end():
    """base_quadrotor_with_gimbal_camera_imu at 1,024 envs: builds through SimBuilder, publishes imu_measurement every env step; after
    1 s of levelled banked flight the camera IMU's gyro reads a link at rest and its accelerometer the thrust's specific force"""
    from aerial_gym_simulator_b200.sim.sim_builder import SimBuilder
    from tests.test_articulated_body_state_cpu import gimbal_levelling
    n = 1024 if DEV != "cpu" else 4
    torch.manual_seed(0)
    env = SimBuilder().build_env("base_sim", "empty_env", "base_quadrotor_with_gimbal_camera_imu", "lee_attitude_control", DEV,
                                 args={"seed": 4}, num_envs=n)
    gtd = env.global_tensor_dict
    assert env.engine.imu_body == gtd["robot_body_names"].index("pitch_stage_link")
    before = gtd["imu_measurement"].clone()
    env.step(torch.zeros(n, 4, device=DEV))
    env.render()
    assert not torch.equal(before, gtd["imu_measurement"])
    gimbal_levelling(env, 100, DEV)
    env.render()
    m = gtd["imu_measurement"].double().cpu()
    assert torch.isfinite(m).all()
    assert m[:, 3:6].abs().max() < 0.1
    assert ((m[:, 0:3].norm(dim=1) - 9.81).abs() < 0.5).all()
