"""Prismatic joints of articulated robots on the H100: agx_hp1_articulated_step_prismatic in its four instantiations on trees mixing
revolute, continuous and prismatic joints against the host shadow and the float64 oracle, the base's momentum balance on the device,
a revolute-only tree through the new kernel against the plain kernel, CUDA-graph step mode against launch mode with the IMU, effort
and joint forces on, agx_hp1_articulated_body_state_prismatic against the oracle, and a camera on the sliding payload.  With
--gpu-dryrun the same text runs on the host shadow (tests/_cpu_stack_articulated_prismatic.py)."""
import contextlib

import numpy as np
import pytest
import torch

from aerial_gym_simulator_b200.hp1 import Hp1Engine
from oracle import articulated_prismatic_oracle as PO
from tests import _hp1_common as H
from tests._cpu_stack_articulated_prismatic import CpuPrismaticHp1Engine, prismatic_twin_for_dryrun
from tests.test_articulated_body_state_cpu import _oracle_image
from tests.test_articulated_cpu import load_inputs, morphy_compliant, random_root, substep_inputs
from tests.test_articulated_imu_cpu import _depth, _limit_crossing
from tests.test_articulated_prismatic_cpu import ROBOT, check_all, mixed_art, ptable, quad_slider

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
STATE = ("root_state", "motor_thrust", "dof_state") + Hp1Engine.DERIVED
EPS = float(np.finfo(np.float32).eps)


@pytest.fixture(autouse=True)
def _twin():
    with prismatic_twin_for_dryrun() if DEV == "cpu" else contextlib.nullcontext():
        yield


def _engine(spec, n, art, imu_body=None, dev=None, joint_force=True):
    dev = DEV if dev is None else dev
    if dev == "cpu":
        return CpuPrismaticHp1Engine(spec, n, per_env_params="all", articulation=art, imu_body=imu_body, joint_force=joint_force)
    return Hp1Engine(spec, n, dev, per_env_params="all", articulation=art, imu_body=imu_body, joint_force=joint_force)


def _step(eng, inp, effort=None, steps=1):
    load_inputs(eng, inp)
    dev = eng.root_state.device
    if eng.dof_actuation_force is not None:
        eng.dof_actuation_force.copy_(effort.to(dev))
    eng.physics_step(inp["actions"].to(dev), disturbance=inp["dist"].to(dev), physics_steps=steps)
    if DEV != "cpu":
        torch.cuda.synchronize()


@pytest.mark.parametrize("M", [4, 8])
@pytest.mark.parametrize("B", [1, 2, 9, 10, 16])
def test_kernel_matches_shadow_and_oracle(M, B):
    """every instantiation <M, 9 | 16> on a mixed tree with effort DOFs, the IMU on its last body, joint forces on at odd N and off
    at the others, on 32 envs spread over the grid: state, IMU input and joint forces within the float64 bars of check_all (the
    dof_force identity on the device's own outputs included).  Against the shadow, every env within 1e-3 of each quantity's largest
    magnitude over the grid (the two differ by the device's FMA contraction, as in the joint-force kernel's test)."""
    rng = np.random.default_rng(2200 + 10 * B + M)
    spec = H.spec_for("quad_attitude" if M == 4 else "octa_velocity")
    art = mixed_art(rng, B, M=M, effort=True)
    b = B - 1
    for N in ((1, 127, 129, 4097, 65536) if DEV != "cpu" else (1, 127, 129)):
        inp = substep_inputs(spec, art, N, 5000 + N + B)
        if N == 129:
            inp = _limit_crossing(inp, art)
        effort = torch.tensor(rng.uniform(-0.6, 0.6, (N, B - 1)), dtype=torch.float32)
        jf = N % 2 == 1 or B == 1
        eng = _engine(spec, N, art, b, joint_force=jf)
        _step(eng, inp, effort)
        sh = _engine(spec, N, art, b, dev="cpu", joint_force=jf)
        _step(sh, inp, effort)
        keys = STATE + ("imu_input",) + (("joint_wrench", "dof_force") if jf else ())
        for k in keys:
            x, y = getattr(eng, k).cpu(), getattr(sh, k)
            r = 0.0 if x.numel() == 0 else float((x - y).abs().max() / (y.abs().max() + 1e-6))
            assert r <= 1e-3, (N, k, r)
        idx = np.unique(np.linspace(0, N - 1, min(N, 32)).astype(int))
        check_all(eng, spec, art, inp, idx, b, effort if art.effort_dof.any() else None)


def test_base_momentum_balance_on_the_device():
    """the sliding-payload quadrotor at 4,096 envs: the base's Newton-Euler balance from the device's rows -- thrusts, drag,
    disturbance and gravity on the base minus what the rail joint takes equals the base's rate of momentum m_0 a_c,0 (the IMU's
    force input on body 0) -- within the float32 error of the rows"""
    from oracle import articulated_imu_oracle as IO
    from oracle import articulated_joint_force_oracle as JO
    from tests.test_articulated_cpu import oracle_state
    spec = H.spec_for("quad_attitude")
    _, art = quad_slider()
    N = 4096 if DEV != "cpu" else 64
    inp = substep_inputs(spec, art, N, 77)
    eng = _engine(spec, N, art, imu_body=0)
    _step(eng, inp)
    W = eng.joint_wrench.cpu().double().numpy()
    f0 = eng.imu_input.cpu().double().numpy()[:, 0:3]
    table = ptable(eng.art, art.prismatic_mask())
    model, st = oracle_state(eng, spec, inp, np.arange(N))
    ok = H.well_conditioned(model, st, inp["actions"].double()).numpy()
    thrust, F_w, _ = IO.substep_inputs(model, st, inp["actions"].double(), inp["dist"].double())
    dof = inp["dof"].double().numpy()
    worst = 0.0
    for n in np.flatnonzero(ok)[:: max(1, N // 512)]:
        R, P = PO.newton_euler(table, st.root[n].numpy(), dof[n, :, 0], dof[n, :, 1], np.zeros(6), np.zeros(1), model.gravity, thrust[n],
                               F_w[n], np.zeros(3))[1:]
        fext = JO.external_forces(table, R, P, np.zeros(3), thrust[n], F_w[n], np.zeros(3))[0, 3:]
        err = np.abs(R[0] @ f0[n] - (fext - R[1] @ W[n, 1, 0:3])).max()
        worst = max(worst, err / (np.abs(thrust[n]).sum() + 9.81 * table["mass"].sum()))
    assert worst <= 1e-4, worst


def test_revolute_tree_through_the_new_kernel_matches_the_plain_kernel():
    """morphy_compliant (no prismatic joint) through agx_hp1_articulated_step_prismatic with prismatic_mask 0 against
    agx_hp1_articulated_step: separate compilations, so the state after 3 sub-steps agrees to float32 rounding"""
    spec = H.spec_for("quad_attitude")
    _, art = morphy_compliant()
    N = 4097 if DEV != "cpu" else 64
    inp = substep_inputs(spec, art, N, 5)
    a, p = _engine(spec, N, art, joint_force=False), _engine(spec, N, art, joint_force=False)
    _step(p, inp, steps=3)
    dev = a.root_state.device
    # physics_step points the buffers at these tensors, and the direct launch below reads them: they must outlive it
    actions, dist = inp["actions"].to(dev), inp["dist"].to(dev)
    load_inputs(a, inp)
    a.physics_step(actions, disturbance=dist, physics_steps=3)
    load_inputs(a, inp)  # again, from the same start, through the prismatic entry
    if DEV != "cpu":
        from aerial_gym_simulator_b200 import _lib
        _lib.check(a.lib.agx_hp1_articulated_step_prismatic(a._cfg_ref, a._buf_ref, a._art_ref, 0, None, 0, None, None, None, a._stream()),
                   "agx_hp1_articulated_step_prismatic")
        torch.cuda.synchronize()
    else:
        from tests import _articulated_prismatic_shadow
        assert _articulated_prismatic_shadow.load().shadow_art_step_prismatic(a._cfg_ref, a._buf_ref, a._art_ref, 0, None, 0, None, None, None) == 0
    for k in STATE:
        x, y = getattr(a, k).cpu(), getattr(p, k).cpu()
        assert ((x - y).abs() / (y.abs().amax(0, keepdim=True) + 1e-6)).max() <= 1e-5, k


def _register(name):
    from aerial_gym_simulator_b200.config import robot_config as rc
    from aerial_gym_simulator_b200.config.sensor_config import BaseImuConfig
    from aerial_gym_simulator_b200.registry._core import robot_registry
    from aerial_gym_simulator_b200.robots import ArticulatedMultirotor
    base = rc.BaseQuadWithSlidingPayloadCfg

    class Cfg(base):
        class joint_config(base.joint_config):
            drive_mode = "effort"
            enable_dof_force_sensors = True

        class sensor_config(base.sensor_config):
            enable_imu = True

            class imu_config(BaseImuConfig):
                parent_link = "payload_link"
    robot_registry.register(name, ArticulatedMultirotor, Cfg)
    return name


def test_graph_step_mode_is_bit_identical_to_launch_mode():
    """20 env steps of the sliding payload in effort mode with an IMU on payload_link and the joint forces on, in env_with_obstacles
    (its scene puts the env step on the graph path), new forces each step and resets of every fifth env every fifth step"""
    from aerial_gym_simulator_b200.env_manager.env_manager import EnvManager
    name = _register("_test_sliding_payload_effort_imu_jf")
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
        f = (torch.rand(n, 1, generator=g) * 2 - 1) * 1.5  # beyond the 1 N limit half the time
        for env in envs.values():
            env.global_tensor_dict["dof_actuation_force_tensor"].copy_(f.to(DEV))
            env.step(a.to(DEV))
            if k % 5 == 4:
                torch.manual_seed(k)
                env.reset_idx(torch.arange(k % 5, n, 5, device=DEV))
        gg, gl = envs["graph"].global_tensor_dict, envs["launch"].global_tensor_dict
        for key in ("dof_force_tensor", "robot_joint_wrench_tensor", "dof_state_tensor", "robot_state_tensor", "robot_body_state_tensor"):
            assert torch.equal(gg[key], gl[key]), (k, key)
        assert torch.equal(envs["graph"].engine.imu_input, envs["launch"].engine.imu_input), k
    assert (gg["dof_state_tensor"][:, 0, 0] != 0).any() and (gg["dof_force_tensor"] != 0).any()
    if DEV != "cpu":
        assert envs["graph"].step_mode == "graph" and envs["graph"]._graphs


@pytest.mark.parametrize("B", [2, 9, 10, 16])
def test_body_states_match_oracle(B):
    """agx_hp1_articulated_body_state_prismatic at N = 4,097 (8 envs checked against the float64 oracle with the bar of the CPU
    test, every env against the shadow within 1e-5 of the row's magnitude)"""
    rng = np.random.default_rng(900 + B)
    spec = H.spec_for("quad_attitude")
    art = mixed_art(rng, B)
    N = 4097 if DEV != "cpu" else 64
    inp = substep_inputs(spec, art, N, 31 + B)
    eng, sh = _engine(spec, N, art, joint_force=False), _engine(spec, N, art, dev="cpu", joint_force=False)
    for e in (eng, sh):
        load_inputs(e, inp)
        e.update_body_state()
    if DEV != "cpu":
        torch.cuda.synchronize()
    got, ref_sh = eng.body_state.cpu(), sh.body_state
    assert torch.equal(got[:, 0], inp["root"])
    assert ((got - ref_sh).abs() / (ref_sh.abs().amax(0, keepdim=True) + 1.0)).max() <= 1e-5
    t = ptable(eng.art, art.prismatic_mask())
    for k in np.unique(np.linspace(0, N - 1, 8).astype(int)):
        ref = PO.body_states(t, inp["root"][k].double().numpy(), inp["dof"][k, :, 0].double().numpy(), inp["dof"][k, :, 1].double().numpy())
        g = got[k].double().numpy()
        for i in range(1, B):
            e = 32 * EPS * (_depth(t, i) + 1)
            qs = ref[i, 3:7] if ref[i, 3:7] @ g[i, 3:7] >= 0 else -ref[i, 3:7]
            assert np.abs(g[i, 0:3] - ref[i, 0:3]).max() <= e * (np.abs(ref[i, 0:3] - ref[0, 0:3]).max() + 1.0) + 4 * EPS * np.abs(ref[i, 0:3]).max()
            assert np.abs(g[i, 3:7] - qs).max() <= e
            assert np.abs(g[i, 7:13] - ref[i, 7:13]).max() <= e * (np.abs(ref[i, 7:13]).max() + np.abs(ref[:, 10:13]).max() + 1.0)


def test_camera_on_the_sliding_payload():
    """a depth camera on payload_link in an obstacle env, the payload driven to setpoints across its rail: the image equals the
    brute-force oracle's at the pose published for the payload's body, bit for bit"""
    from aerial_gym_simulator_b200.config import robot_config as rc
    from aerial_gym_simulator_b200.config.sensor_config import GimbalDepthCameraConfig
    from aerial_gym_simulator_b200.env_manager.env_manager import EnvManager
    from aerial_gym_simulator_b200.registry._core import robot_registry
    from aerial_gym_simulator_b200.robots import ArticulatedMultirotor
    base = rc.BaseQuadWithSlidingPayloadCfg

    class Cam(GimbalDepthCameraConfig):
        parent_link = "payload_link"

    class Cfg(base):
        class sensor_config(base.sensor_config):
            enable_camera = True
            camera_config = Cam
    robot_registry.register("_test_sliding_payload_camera", ArticulatedMultirotor, Cfg)
    n = 1024 if DEV != "cpu" else 4
    torch.manual_seed(0)
    env = EnvManager("base_sim", "env_with_obstacles", "_test_sliding_payload_camera", "lee_attitude_control", DEV, num_envs=n,
                     args={"seed": 4})
    env.reset()
    gtd = env.global_tensor_dict
    gtd["dof_position_setpoint_tensor"][:, 0] = torch.linspace(-0.05, 0.05, n, device=DEV)
    for _ in range(5):
        env.step(torch.zeros(n, 4, device=DEV))
    env.render()
    if DEV != "cpu":
        torch.cuda.synchronize()
    b = gtd["robot_body_names"].index("payload_link")
    assert env.robot.bodies.link_body["payload_link"] == b == 1
    q = gtd["dof_state_tensor"][:, 0, 0].cpu()
    assert q.min() < -0.005 and q.max() > 0.005  # the payloads sit at different places on their rails
    idx = np.unique(np.linspace(0, n - 1, min(n, 24)).astype(int))
    pose = gtd["robot_body_state_tensor"][:, b, :7].cpu().numpy()
    pix, seg = _oracle_image(env, pose, env.sensor_mount.cpu().numpy(), idx)
    assert np.array_equal(gtd["depth_range_pixels"].cpu().numpy()[idx], pix)
    assert np.array_equal(gtd["segmentation_pixels"].cpu().numpy()[idx], seg)
    assert (pix < 1.0).any()
