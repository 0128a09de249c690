"""LiDARNavigationTask epilogue on the GPU, through the C ABI: the three kernels of lidar_nav.cu against (a) the
fixtures produced by the reference's own code and (b) the oracle on bigger random inputs and ragged image shapes; plus
LiDARNavigationTask end to end (env_with_lidar_nav_obstacles: 91 boxes, magpie, 48 x 120 world-frame point cloud).

(Named test_zz_*: these kernels were written after the round's GPU budget was spent -- their arithmetic and indexing
are verified on CPU by tests/test_lidar_nav_cpu.py through the host shadow build -- so they run after every test that
has already been green on a GPU.)"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from aerial_gym_simulator_b200 import _lib
from oracle import hp1_oracle as O
from oracle import lidar_nav_oracle as L

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden", "lidar_nav_task_epilogue.npz")
DEV = "cuda:0"


def _d(x, dtype=torch.float32):
    return torch.tensor(np.asarray(x), dtype=dtype, device=DEV).contiguous()


def _p(t):
    return C.c_void_p(t.data_ptr())


def _params(d):
    assert tuple(d["param_names"]) == L.LIDAR_NAV_PARAM_NAMES
    p = _lib.AgxLidarNavRewardParams()
    for i, v in enumerate(d["param_values"]):
        p.v[i] = float(v)
    return p, {k: float(v) for k, v in zip(d["param_names"], d["param_values"])}


def _pool_gpu(pc, pos, vel, ph=3, pw=6, offset_floats=0):
    """pc [N,H,W,3] (cpu); offset_floats shifts the cloud inside its allocation (exercises the non-16-byte-aligned path)."""
    lib = _lib.load()
    n, H, W, _ = pc.shape
    raw = torch.zeros(pc.numel() + 8, device=DEV)
    pcd = raw[offset_floats:offset_floats + pc.numel()].view(n, H, W, 3)
    pcd.copy_(pc.to(DEV))
    st = torch.zeros(n, 13, device=DEV)
    st[:, 0:3], st[:, 7:10], st[:, 6] = pos.to(DEV), vel.to(DEV), 1.0
    ds = torch.full((n, H // ph, W // pw), -7.0, device=DEV)
    ttc = torch.full((n,), -7.0, device=DEV)
    _lib.check(lib.agx_lidar_nav_pool(n, H, W, ph, pw, _p(pcd), _p(st), 13, 10.0, 0.2, 10.0, 10.0, _p(ds), _p(ttc), None), "agx_lidar_nav_pool")
    torch.cuda.synchronize()
    return ds.cpu(), ttc.cpu()


@pytest.mark.parametrize("offset", [0, 1])
def test_pool_kernel_matches_reference_fixture(offset):
    d = np.load(G)
    ds, ttc = _pool_gpu(torch.tensor(d["pool_pointcloud"]), torch.tensor(d["pool_robot_position"]), torch.tensor(d["pool_robot_linvel"]),
                        offset_floats=offset)
    ref = torch.tensor(d["pool_image_ds"])
    assert torch.allclose(ds, ref, rtol=1e-6, atol=0), (ds - ref).abs().max()
    assert torch.equal(ds == 10.0, ref == 10.0)  # clipping decisions agree exactly
    assert torch.allclose(ttc, torch.tensor(d["pool_time_to_collision"]), rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("n,H,W,ph,pw", [(300, 48, 120, 3, 6), (5, 7, 13, 3, 6), (5, 5, 9, 2, 2), (3, 1, 40, 1, 7), (4, 64, 33, 4, 3),
                                          (2, 3, 6, 3, 6), (2, 128, 512, 2, 8)])  # the last one: 96 KB of band staging, the > 48 KB opt-in path
def test_pool_kernel_matches_oracle_any_shape(n, H, W, ph, pw):
    g = torch.Generator().manual_seed(H * 1000 + W)
    pos = torch.randn(n, 3, generator=g)
    vel = torch.randn(n, 3, generator=g) * 2
    vel[0] = 0.0
    dirs = torch.randn(n, H, W, 3, generator=g)
    dirs = dirs / dirs.norm(dim=-1, keepdim=True)
    rng = torch.rand(n, H, W, 1, generator=g) * 13 + 0.05
    rng = torch.where((rng - 10.0).abs() < 1e-3, rng + 0.01, rng)  # 1 ulp must not decide a clipping
    rng = torch.where((rng - 0.2).abs() < 1e-3, rng + 0.01, rng)
    pc = pos.view(n, 1, 1, 3) + dirs * rng
    want_ds, want_ttc = L.pool(pc, pos, vel, (ph, pw))
    ds, ttc = _pool_gpu(pc, pos, vel, ph, pw)
    assert torch.allclose(ds, want_ds, rtol=1e-6, atol=0), (ds - want_ds).abs().max()
    assert torch.allclose(ttc, want_ttc, rtol=1e-4, atol=1e-5), (ttc - want_ttc).abs().max()
    assert float(ttc[0]) == 10.0


def _reward_gpu(a, frac, params):
    lib, n = _lib.load(), a["pos"].shape[0]
    state = torch.zeros(n, 13, device=DEV)
    state[:, 0:3] = _d(a["pos"])
    t = [_d(a[k]) for k in ("vehicle_orientation", "target", "euler", "target_yaw", "vehicle_linvel", "body_angvel")]
    t.append(_d(np.asarray(a["crashes"]), torch.uint8))
    t += [_d(a[k]) for k in ("actions", "prev_actions", "time_to_collision")]
    pe, pp, rew = _d(a["prev_pos_error"]).clone(), torch.zeros(n, 3, device=DEV), torch.zeros(n, device=DEV)
    _lib.check(lib.agx_lidar_nav_reward(n, _p(state), 13, *[_p(x) for x in t], float(frac), C.byref(params), _p(pe), _p(pp), _p(rew), None),
               "agx_lidar_nav_reward")
    torch.cuda.synchronize()
    return rew.cpu(), pe.cpu(), pp.cpu()


@pytest.mark.parametrize("tag", ["c0", "c1"])
def test_reward_kernel_matches_reference_fixture(tag):
    d = np.load(G)
    params, _ = _params(d)
    rew, pe, pp = _reward_gpu(d, d[f"frac_{tag}"], params)
    ref = torch.tensor(d[f"reward_{tag}"])
    assert torch.allclose(rew, ref, rtol=1e-5, atol=1e-4), (rew - ref).abs().max()
    assert torch.allclose(pe, torch.tensor(d["pos_error"]), rtol=1e-5, atol=1e-5)
    assert torch.equal(pp, torch.tensor(d["prev_pos_error"]))
    assert torch.equal(rew[::11], torch.full_like(rew[::11], -10.0))


def test_reward_kernel_matches_oracle_on_random_inputs():
    g = torch.Generator().manual_seed(78)
    n = 20001
    r = lambda *s: torch.randn(*s, generator=g)
    q = r(n, 4)
    q = q / q.norm(dim=1, keepdim=True)
    a = {"pos": r(n, 3) * 4, "target": r(n, 3) * 4, "vehicle_orientation": O.vehicle_frame_quat_from_quat(q),
         "euler": torch.rand(n, 3, generator=g) * 2 * np.pi, "target_yaw": (torch.rand(n, generator=g) * 2 - 1) * np.pi,
         "vehicle_linvel": r(n, 3) * 2, "body_angvel": r(n, 3), "crashes": torch.rand(n, generator=g) < 0.05,
         "actions": torch.rand(n, 4, generator=g) * 2 - 1, "prev_actions": torch.rand(n, 4, generator=g) * 2 - 1,
         "time_to_collision": torch.rand(n, generator=g) * 10, "prev_pos_error": r(n, 3)}
    a["target"][:500] = a["pos"][:500] + 0.4 * r(500, 3)
    params, p = _params(np.load(G))
    want, err = L.rewards_and_errors(a["vehicle_orientation"], a["pos"], a["target"], a["euler"], a["target_yaw"], a["vehicle_linvel"],
                                     a["body_angvel"], a["crashes"], a["actions"], a["prev_actions"], a["time_to_collision"], 0.6, p)
    rew, pe, _ = _reward_gpu({k: v.numpy() for k, v in a.items()}, 0.6, params)
    assert torch.allclose(rew, want, rtol=1e-5, atol=2e-4), (rew - want).abs().max()
    assert torch.allclose(pe, err, rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("obs_stride,num_lidar", [(337, 320), (400, 320), (17, 0)])
def test_obs_kernel_matches_reference_fixture(obs_stride, num_lidar):
    d = np.load(G)
    lib, n = _lib.load(), d["pos"].shape[0]
    state = torch.zeros(n, 13, device=DEV)
    state[:, 0:3] = _d(d["pos"])
    t = [_d(d[k]) for k in ("vehicle_orientation", "euler", "body_linvel", "body_angvel", "robot_actions", "target", "target_yaw",
                            "obs_draw_vec", "obs_draw_euler")]
    lidar = _d(d["obs"][:, 17:17 + num_lidar]) if num_lidar else None
    obs = torch.full((n, obs_stride), 7.0, device=DEV)
    _lib.check(lib.agx_lidar_nav_obs(n, _p(state), 13, *[_p(x) for x in t], _p(lidar) if num_lidar else None, num_lidar, _p(obs), obs_stride,
                                     None), "agx_lidar_nav_obs")
    torch.cuda.synchronize()
    ref = torch.tensor(d["obs"])[:, :17 + num_lidar]
    got = obs.cpu()
    assert torch.allclose(got[:, :17 + num_lidar], ref, rtol=1e-5, atol=1e-5), (got[:, :17 + num_lidar] - ref).abs().max()
    assert torch.equal(got[:, 17:17 + num_lidar], ref[:, 17:])  # the LiDAR columns are a copy
    assert (got[:, 17 + num_lidar:] == 7.0).all()


def test_argument_validation():
    lib = _lib.load()
    x = torch.zeros(64, device=DEV)
    assert lib.agx_lidar_nav_pool(1, 4, 4, 5, 2, _p(x), _p(x), 13, 10.0, 0.2, 10.0, 10.0, _p(x), _p(x), None) == -1  # pool_h > height
    assert lib.agx_lidar_nav_pool(1, 4, 4, 2, 2, _p(x), _p(x), 9, 10.0, 0.2, 10.0, 10.0, _p(x), _p(x), None) == -1   # stride < 10
    assert lib.agx_lidar_nav_pool(1, 4, 4, 2, 2, None, _p(x), 13, 10.0, 0.2, 10.0, 10.0, _p(x), _p(x), None) == -3
    assert lib.agx_lidar_nav_pool(0, 4, 4, 2, 2, None, None, 13, 10.0, 0.2, 10.0, 10.0, None, None, None) == 0       # empty batch
    assert lib.agx_lidar_nav_pool(1, 64, 4096, 8, 8, _p(x), _p(x), 13, 10.0, 0.2, 10.0, 10.0, _p(x), _p(x), None) == -1  # band > smem
    assert b"shared memory" in lib.agx_last_error()


def test_lidar_navigation_task_end_to_end():
    """task_registry.make_task('lidar_navigation_task'): reset, a few steps, and every stage of the epilogue against the
    oracle fed with the task's own tensors."""
    import aerial_gym_simulator_b200.task  # noqa: F401
    from aerial_gym_simulator_b200.registry._core import task_registry

    N = 12
    task = task_registry.make_task("lidar_navigation_task", seed=7, num_envs=N, headless=True)
    od = task.obs_dict
    assert od["depth_range_pixels"].shape == (N, 1, 48, 120, 3) and od["num_obstacles_in_env"] == 25  # curriculum min level
    assert task.sim_env.scene.K >= 91  # 15 panels + 70 objects + 6 walls, one box each
    obs, rew, term, trunc, info = task.reset()
    assert obs["observations"].shape == (N, 337)
    assert (obs["observations"][:, 17:] == 0).all()  # no LiDAR frame processed yet (downsampled_lidar_data starts at zero)
    assert (task.target_yaw.abs() <= np.pi).all()
    g = torch.Generator(device=DEV).manual_seed(0)
    for _ in range(4):
        a = (torch.rand(N, 4, device=DEV, generator=g) * 2 - 1) * 0.3
        out = task.step(a)
        assert out[0] is obs and out[1] is rew
    torch.cuda.synchronize()
    assert torch.isfinite(obs["observations"]).all() and torch.isfinite(rew).all()
    assert torch.equal(obs["observations"][:, 17:], task.downsampled_lidar_data)
    assert (task.time_to_collision >= 0).all() and (task.time_to_collision <= 10).all()
    assert torch.allclose(task.current_action[:, 0:3], 2 * a[:, 0:3]) and torch.equal(obs["observations"][:, 13:17], od["robot_actions"])
    # the pooling stage against the oracle, on the frame the task holds (noise switched off for the comparison)
    task.add_noise_to_downsampled_lidar_data = lambda x: x
    task.process_image_observation()
    torch.cuda.synchronize()
    pc = od["depth_range_pixels"].squeeze(1).cpu()
    want_ds, want_ttc = L.pool(pc, od["robot_position"].cpu(), od["robot_linvel"].cpu())
    got_ds = task._image_ds.cpu()
    r = (pc - od["robot_position"].cpu().view(N, 1, 1, 3)).norm(dim=-1)
    near = ((r - 10.0).abs().lt(1e-4) | (r - 0.2).abs().lt(1e-5)).view(N, 16, 3, 20, 6).any(4).any(2)
    ok = torch.isclose(got_ds, want_ds, rtol=1e-5, atol=0) | near  # a return within 0.1 mm of a clipping threshold may fall either way
    assert ok.all(), (got_ds - want_ds).abs().max()
    assert torch.allclose(task.time_to_collision.cpu(), want_ttc, rtol=1e-4, atol=1e-5)
    assert torch.allclose(task.downsampled_lidar_data.cpu(), (1 / got_ds).view(N, -1), rtol=1e-6, atol=0)
    assert (got_ds >= 0.2 - 1e-6).all() and (got_ds <= 10.0).all()
    # the reward stage against the oracle
    params, p = _params(np.load(G))
    prev_err = task.pos_error_vehicle_frame.cpu().clone()
    task.compute_rewards_and_crashes(od)
    torch.cuda.synchronize()
    want, err = L.rewards_and_errors(od["robot_vehicle_orientation"].cpu(), od["robot_position"].cpu(), task.target_position.cpu(),
                                     od["robot_euler_angles"].cpu(), task.target_yaw.cpu(), od["robot_vehicle_linvel"].cpu(),
                                     od["robot_body_angvel"].cpu(), od["crashes"].cpu(), task.current_action.cpu(), task.prev_action.cpu(),
                                     task.time_to_collision.cpu(), task.curriculum_progress_fraction, p)
    assert torch.allclose(task.rewards.cpu(), want, rtol=1e-5, atol=2e-4), (task.rewards.cpu() - want).abs().max()
    assert torch.allclose(task.pos_error_vehicle_frame.cpu(), err, rtol=1e-5, atol=1e-5)
    assert torch.equal(task.pos_error_vehicle_frame_prev.cpu(), prev_err)
    # the observation stage against the oracle, with given draws
    u1, u2 = torch.rand(N, 3, device=DEV), torch.rand(N, 3, device=DEV)
    task.process_obs_for_task(u1, u2)
    torch.cuda.synchronize()
    want_obs = L.process_obs(od["robot_vehicle_orientation"].cpu(), od["robot_position"].cpu(), task.target_position.cpu(),
                             od["robot_euler_angles"].cpu(), task.target_yaw.cpu(), od["robot_body_linvel"].cpu(), od["robot_body_angvel"].cpu(),
                             od["robot_actions"].cpu(), task.downsampled_lidar_data.cpu(), u1.cpu(), u2.cpu())
    assert torch.allclose(obs["observations"].cpu(), want_obs, rtol=1e-5, atol=1e-5)
    task.close()


@pytest.mark.parametrize("tag", ["c0", "c1"])
def test_radar_variant_reward_kernel_matches_reference_fixture(tag):
    """RadarNavigationTask's compute_reward (one term differs from the LiDAR task's)"""
    d = np.load(G)
    params, _ = _params(d)
    params.radar_variant = 1
    rew, _, _ = _reward_gpu(d, d[f"frac_{tag}"], params)
    ref = torch.tensor(d[f"radar_reward_{tag}"])
    assert torch.allclose(rew, ref, rtol=1e-5, atol=1e-4), (rew - ref).abs().max()


def test_radar_navigation_task_end_to_end():
    import aerial_gym_simulator_b200.task  # noqa: F401
    from aerial_gym_simulator_b200.registry._core import task_registry

    N = 8
    task = task_registry.make_task("radar_navigation_task", seed=9, num_envs=N, headless=True)
    od = task.obs_dict
    assert od["depth_range_pixels"].shape == (N, 1, 48, 120, 3) and task._params.radar_variant == 1
    obs, rew, term, trunc, info = task.reset()
    for _ in range(3):
        obs, rew, term, trunc, info = task.step(torch.rand(N, 4, device=DEV) * 0.6 - 0.3)
    torch.cuda.synchronize()
    ds = task.downsampled_lidar_data
    assert torch.isfinite(ds).all() and 0.6 < float((ds == -1.0).float().mean()) < 0.95
    assert torch.equal(obs["observations"][:, 17:], ds) and torch.isfinite(rew).all()
    _, p = _params(np.load(G))
    task.compute_rewards_and_crashes(od)
    torch.cuda.synchronize()
    c = lambda t: t.cpu()
    want, _ = L.rewards_and_errors(c(od["robot_vehicle_orientation"]), c(od["robot_position"]), c(task.target_position), c(od["robot_euler_angles"]),
                                   c(task.target_yaw), c(od["robot_vehicle_linvel"]), c(od["robot_body_angvel"]), c(od["crashes"]),
                                   c(task.current_action), c(task.prev_action), c(task.time_to_collision), task.curriculum_progress_fraction, p,
                                   radar_variant=True)
    assert torch.allclose(c(task.rewards), want, rtol=1e-5, atol=2e-4)
    task.close()
