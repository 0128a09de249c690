"""Per-body state of articulated robots on the H100: agx_hp1_articulated_body_state against the float64 body_states() of
oracle/articulated_body_state_oracle.py and its host shadow, CUDA-graph step mode against launch mode for robot_body_state_tensor, and the gimbal
quadrotor's camera and levelling in an obstacle env.  With --gpu-dryrun the same text runs on the host shadow
(tests/_cpu_stack_articulated.py)."""
import contextlib
import ctypes as C

import numpy as np
import pytest
import torch

from aerial_gym_simulator_b200 import _lib
from tests import _articulated_shadow
from tests._cpu_stack_articulated import articulated_twin_for_dryrun
from tests.test_articulated_body_state_cpu import _cases, _check_rows, gimbal_camera_check, levelling_check
from tests.test_articulated_cpu import morphy_compliant, random_art, table_of

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(autouse=True)
def _body_state_twin():
    """with --gpu-dryrun (tests/conftest.py has set DEV to "cpu" and entered the CPU stack) EnvManager's engine is the CPU twin that
    publishes the body states; on the GPU nothing changes"""
    with articulated_twin_for_dryrun() if DEV == "cpu" else contextlib.nullcontext():
        yield


def _launch(art, roots, dof, stride):
    """the entry point on the device (the shadow under --gpu-dryrun) with root rows `stride` floats apart -> body_state [N,B,13]"""
    N = roots.shape[0]
    dof_t = torch.tensor(dof, device=DEV).contiguous()
    root_t = torch.zeros(N, stride, device=DEV)
    root_t[:, :13] = torch.tensor(roots, device=DEV)
    s = art.to_struct()
    s.dof_state = dof_t.data_ptr()
    out = torch.full((N, s.num_bodies, 13), float("nan"), device=DEV)
    if DEV == "cpu":
        _articulated_shadow.body_state(s, root_t, out)
    else:
        lib = _lib.load()
        _lib.check(lib.agx_hp1_articulated_body_state(C.byref(s), N, root_t.data_ptr(), stride, out.data_ptr(),
                                                      torch.cuda.current_stream().cuda_stream), "agx_hp1_articulated_body_state")
        torch.cuda.synchronize()
    return out.cpu().numpy(), s


@pytest.mark.parametrize("B", [1, 2, 9, 10, 16])
def test_kernel_matches_oracle_and_shadow(B):
    """every env: row 0 bit for bit, every row within the tolerance of _check_rows (its derivation) of the host shadow, which differs
    only by the device's FMA contraction; 48 envs spread over each grid, the first and last included: within _check_rows of the
    float64 oracle.  Strided root rows (stride 20) give the same rows as contiguous ones, bit for bit."""
    rng = np.random.default_rng(100 + B)
    art = morphy_compliant()[1] if B == 9 else random_art(rng, B)
    for N in ((1, 127, 129, 4097, 65536) if DEV != "cpu" else (1, 127, 129)):
        roots, dofs = _cases(rng, B, N)
        got, s = _launch(art, roots, dofs, 13)
        strided, _ = _launch(art, roots, dofs, 20)
        assert np.array_equal(got, strided)
        assert np.array_equal(got[:, 0], roots)
        sh = np.zeros_like(got)
        ss = art.to_struct()
        dof_t = torch.tensor(dofs).contiguous()
        ss.dof_state = dof_t.data_ptr()
        sh_t = torch.from_numpy(sh)
        _articulated_shadow.body_state(ss, torch.tensor(roots), sh_t)
        assert np.isfinite(got).all()
        # device vs shadow: positions / velocities by value, rotations as matrices
        d = np.abs(got - sh)
        assert d[..., 0:3].max() <= 1e-4 + 4 * np.finfo(np.float32).eps * np.abs(roots[:, 0:3]).max(), d[..., 0:3].max()
        assert d[..., 7:13].max() <= 1e-3, d[..., 7:13].max()
        table = table_of(s)
        for n in sorted(set(np.linspace(0, N - 1, min(N, 48)).astype(int))):
            _check_rows(table, roots[n].astype(np.float64), dofs[n].astype(np.float64), got[n])


def _env(mode, n):
    from aerial_gym_simulator_b200.env_manager.env_manager import EnvManager
    torch.manual_seed(0)
    env = EnvManager("base_sim", "empty_env", "morphy_compliant", "lee_attitude_control", DEV, num_envs=n,
                     args={"step_mode": mode, "seed": 3})
    env.reset()
    return env


def test_graph_step_mode_body_state_is_bit_identical_to_launch_mode():
    """20 env steps with resets of every fifth env every fifth step (morphy_compliant draws disturbances: the graph path)"""
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
                torch.manual_seed(k)  # the joint-state draw of reset_idx is torch's: the same for both managers
                env.reset_idx(torch.arange(k % 5, n, 5, device=DEV))
        gg, gl = envs["graph"].global_tensor_dict, envs["launch"].global_tensor_dict
        assert torch.equal(gg["robot_body_state_tensor"], gl["robot_body_state_tensor"]), k
    assert torch.equal(gg["robot_body_state_tensor"][:, 0], gg["robot_state_tensor"])
    if DEV != "cpu":
        assert envs["graph"].step_mode == "graph" and envs["graph"]._graphs


def test_gimbal_camera_in_an_obstacle_env():
    from aerial_gym_simulator_b200.env_manager.env_manager import EnvManager
    n = 1024 if DEV != "cpu" else 4
    torch.manual_seed(0)
    env = EnvManager("base_sim", "env_with_obstacles", "base_quadrotor_with_gimbal_camera", "lee_attitude_control", DEV, num_envs=n,
                     args={"seed": 4})
    env.reset()
    gtd = env.global_tensor_dict
    gtd["dof_position_setpoint_tensor"][:, 0] = torch.linspace(-0.6, 0.6, n, device=DEV)
    gtd["dof_position_setpoint_tensor"][:, 1] = torch.linspace(-0.6, 1.5, n, device=DEV)
    for _ in range(3):
        env.step(torch.zeros(n, 4, device=DEV))
    env.render()
    torch.cuda.synchronize()
    idx = np.unique(np.linspace(0, n - 1, min(n, 24)).astype(int))
    pix = gimbal_camera_check(env, idx)
    assert (pix < 1.0).any()
    levelling_check(env, DEV)
