"""Ray-cast sensor noise on the GPU: agx_hp2_noise_limits (device RNG) against the numpy oracle, its distribution against the
reference-order torch path, the unfused (raw) output of agx_hp2_cast it runs on, and EnvManager with a noisy LiDAR in both
RNG modes.

(Named test_zz_*: written after the round's GPU budget was spent; the device code is verified on CPU through the host
shadow build, tests/test_sensor_noise_cpu.py.)"""
import ctypes as C
import os
import types

import numpy as np
import pytest
import torch

from aerial_gym_simulator_b200 import _lib
from aerial_gym_simulator_b200.sensors.noise import DeviceSensorNoise, apply_noise_and_limits_torch, noise_struct
from oracle import hp2_oracle as RO
from oracle import sensor_noise_oracle as SN
from tests import _hp2_common as H

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden", "sensor_noise.npz")
DEV = "cuda:0"
CASES = ["lidar_range", "lidar_pc_sensor", "lidar_pc_world", "camera_depth_nonoise"]


def _cfg(spec):
    st, pc, world, norm, noise, drop = spec[0], spec[1] == "1", spec[2] == "1", spec[3] == "1", spec[4] == "1", float(spec[5])
    nz = types.SimpleNamespace(enable_sensor_noise=noise, std_a=0.00038089, std_b=-0.00343351, std_c=0.01553284, mean_offset=-0.025,
                               pixel_dropout_prob=drop)
    return types.SimpleNamespace(sensor_type=st, return_pointcloud=pc, pointcloud_in_world_frame=world, normalize_range=norm, max_range=10.0,
                                 min_range=0.2, far_out_of_range_value=10.0, near_out_of_range_value=-10.0, sensor_noise=nz)


def _oracle(px, n, seed, frame, first=0):
    return SN.noise_limits(px, n.components, n.enable_noise, n.apply_limits, n.normalize, n.std_a, n.std_b, n.std_c, n.mean_offset,
                           n.pixel_dropout_prob, n.max_range, n.min_range, n.far_out_of_range_value, n.near_out_of_range_value, seed, frame, first)


def _gpu(px, n, seed, frame, first=0):
    t = torch.tensor(np.ascontiguousarray(px, np.float32), device=DEV)
    _lib.check(_lib.load().agx_hp2_noise_limits(C.c_void_p(t.data_ptr()), t.numel() // n.components, first, C.byref(n), seed, frame, None),
               "agx_hp2_noise_limits")
    torch.cuda.synchronize()
    return t.cpu().numpy()


@pytest.mark.parametrize("name", CASES)
def test_noise_kernel_matches_oracle(name):
    d = np.load(G)
    n = noise_struct(_cfg(d[f"{name}_spec"]))
    px = d[f"{name}_in"]
    seed, frame = 0x1234_5678_9ABC_DEF0, 7
    for first in (0, (1 << 33) + 5):
        got, want = _gpu(px, n, seed, frame, first), _oracle(px, n, seed, frame, first)
        ok = np.isclose(got, want, rtol=1e-4, atol=2e-4 * max(1.0, float(np.abs(want).max())))
        if n.enable_noise and n.apply_limits and not ok.all():
            # device logf / cosf are a few ulp from numpy's: a noisy value within that distance of a range limit may legitimately land on
            # the other side of the threshold -- only those values are excused
            pre = SN.noise_limits(px, n.components, True, False, False, n.std_a, n.std_b, n.std_c, n.mean_offset, n.pixel_dropout_prob,
                                  n.max_range, n.min_range, n.far_out_of_range_value, n.near_out_of_range_value, seed, frame, first)
            mag = np.sqrt((pre.reshape(-1, n.components) ** 2).sum(1)) if n.components == 3 else np.abs(pre.reshape(-1))
            tol = 1e-4 * np.maximum(1.0, np.abs(np.asarray(px, np.float32).reshape(-1, n.components)).max(1)) ** 2
            near_limit = (np.abs(mag - n.max_range) < tol) | (np.abs(mag - n.min_range) < tol)
            ok = ok.reshape(-1, n.components).all(1) | near_limit
            assert near_limit.mean() < 1e-3
        assert ok.all(), np.abs(got - want).max()
    if not n.enable_noise:
        assert np.array_equal(_gpu(px, n, seed, frame), d[f"{name}_out"])  # limits + normalisation only: the reference's output, bit for bit
    else:
        a = _gpu(px, n, seed, frame)
        assert np.array_equal(a, _gpu(px, n, seed, frame)) and not np.array_equal(a, _gpu(px, n, seed, frame + 1))
        half = px.reshape(-1, n.components).shape[0] // 2  # sharding invariance
        assert np.array_equal(a.reshape(-1, n.components)[half:], _gpu(px.reshape(-1, n.components)[half:], n, seed, frame, half))


def test_device_rng_noise_distribution_and_grid_stride():
    """2.4 M pixels (more than one grid-stride sweep of 32 CTAs per SM x 256 threads on a 132-SM H100): moments against the closed form and against
    the reference-order torch path on the same input"""
    cfg = _cfg(np.array(["lidar", "0", "0", "0", "1", "0.05"]))
    cfg.near_out_of_range_value = -1.0
    n = noise_struct(cfg)
    P = 2_400_000
    got = _gpu(np.full((P,), 4.0, np.float32), n, 99, 0)
    dropped = got == -1.0
    assert abs(dropped.mean() - 0.05) < 0.001
    std = 0.00038089 * 16 + -0.00343351 * 4 + 0.01553284
    kept = got[~dropped]
    assert abs(kept.mean() - 4.025) < 5 * std / np.sqrt(kept.size) and abs(kept.std() - std) < 0.005 * std
    torch.manual_seed(0)
    ref = apply_noise_and_limits_torch(torch.full((1, 1, 1, P), 4.0, device=DEV), cfg).cpu().numpy().ravel()
    rk = ref[ref != -1.0]
    assert abs(rk.mean() - kept.mean()) < 8 * std / np.sqrt(kept.size) and abs(rk.std() - kept.std()) < 0.005 * std
    want = _oracle(np.full((4096,), 4.0, np.float32), n, 99, 0, P - 4096)  # the tail of the sweep against the oracle
    assert np.allclose(got[-4096:], want, rtol=1e-4, atol=1e-5)


def test_raw_cast_then_device_noise_matches_oracle_chain():
    """a LiDAR with its noise model on: agx_hp2_cast leaves RAW ranges (bit-identical to the oracle's unfused output), then
    DeviceSensorNoise = oracle noise on those ranges"""
    from tests.test_hp2_gpu import build, oracle_cast

    class Noise:
        enable_sensor_noise = True
        std_a, std_b, std_c, mean_offset, pixel_dropout_prob = 0.00038089, -0.00343351, 0.01553284, -0.025, 0.01

    cfg = H.cfg_variant(H.LidarCfg, sensor_noise=Noise, max_range=10.0, min_range=0.2, far_out_of_range_value=10.0,
                        near_out_of_range_value=-10.0)
    sc = H.make_scene(6, 24, seed=5)
    scene, sensor, robot, mount, _ = build(sc, cfg)
    assert sensor.noise_enabled and sensor.c.fuse_epilogue == 0
    sensor.capture()
    torch.cuda.synchronize()
    raw, ref_seg = oracle_cast(sc, cfg, sensor, robot, mount)
    assert np.array_equal(sensor.pixels.cpu().numpy(), raw), "unfused cast output differs from the oracle"
    assert np.array_equal(sensor.seg_pixels.cpu().numpy(), ref_seg)
    assert (raw < 10.0).any()
    noise = DeviceSensorNoise(cfg, sensor.pixels, seed=11, first_pixel=1000)
    noise.apply()
    torch.cuda.synchronize()
    want = _oracle(raw, noise.c, 11, 0, 1000)
    got = sensor.pixels.cpu().numpy().copy()
    miss = raw > 100.0  # a miss (1000 m) has std = 377 m: it lands beyond max range (far value) or below min range (near value) ...
    assert np.allclose(got[~miss], want[~miss], rtol=1e-4, atol=1e-5), np.abs(got - want)[~miss].max()
    clipped = np.isin(got[miss], np.array([1.0, -1.0], np.float32))
    # ... except the ~1 % of the draws that fall inside [min_range, max_range]: those follow the oracle (a 1e-4 relative error of
    # the normal draw on std 377 m is 0.04 m = 0.004 after the normalisation)
    assert clipped.mean() > 0.95 and np.allclose(got[miss][~clipped], want[miss][~clipped], atol=2e-2)
    assert (np.isin(want[miss], np.array([1.0, -1.0], np.float32)) != clipped).mean() < 1e-3  # same side of the limits as the oracle
    assert (got <= 1.0).all() and (got >= -1.0).all()
    assert noise.frame == 1
    sensor.capture()
    noise.apply()
    torch.cuda.synchronize()
    assert not np.array_equal(sensor.pixels.cpu().numpy(), got)  # next frame, next stream


@pytest.mark.parametrize("mode", ["device", "torch"])
def test_env_manager_noisy_lidar(mode):
    """base_quadrotor_with_lidar carries BaseLidarConfig, whose noise model is ON (base_lidar_config.py:58-64)"""
    import aerial_gym_simulator_b200.task  # noqa: F401
    from aerial_gym_simulator_b200.sim import SimBuilder

    N = 4
    args = {"seed": 3, "sensor_noise_rng": mode} if mode == "device" else {"seed": 3, "reset_rng": "torch"}
    env = SimBuilder().build_env("base_sim", "env_with_obstacles", "base_quadrotor_with_lidar", "lee_velocity_control", DEV, args=args,
                                 num_envs=N, use_warp=True, headless=True)
    assert env.sensor.noise_enabled and env.sensor_noise_rng == mode and (env._device_noise is not None) == (mode == "device")
    env.reset()
    gtd = env.get_obs()
    torch.manual_seed(5)
    env.render()
    torch.cuda.synchronize()
    px = gtd["depth_range_pixels"].clone()
    assert px.shape == (N, 1, 128, 512) and torch.isfinite(px).all() and (px <= 1.0).all() and (px >= -1.0).all()
    # the same frame from the oracle: raw ranges, then the mode's noise
    sc = env.scene
    tris, segs, cnt = RO.build_world_tris(env._obj_pose.cpu().numpy(), sc.obj_template.cpu().numpy(), sc.obj_seg_counter.cpu().numpy(),
                                          sc.tmpl_tri_offset.cpu().numpy(), sc.tmpl_tris.cpu().numpy(), sc.tmpl_seg_base.cpu().numpy(),
                                          sc.tmpl_seg_mask.cpu().numpy(), sc.K * sc.L)
    so, _ = H.oracle_sensor(env.sensor_cfg, fuse=False)
    raw, _ = RO.cast(so, gtd["robot_state_tensor"][:, :7].cpu().numpy(), env.sensor_mount.cpu().numpy(), env.sensor.ray_table.cpu().numpy(),
                     tris, segs, cnt)
    hit = raw < 999.0
    if mode == "device":
        want = _oracle(raw, env._device_noise.c, env._device_noise.seed, 0, 0)
        assert np.allclose(px.cpu().numpy()[hit], want[hit], rtol=1e-4, atol=1e-5)
    else:
        t = torch.tensor(raw, device=DEV)
        torch.manual_seed(5)
        apply_noise_and_limits_torch(t, env.sensor_cfg)
        assert torch.equal(px, t)  # torch path: same seed, same draws
    # BaseLidarConfig: std ~ 1e-5 m, mean offset +0.05 m -> a hit at range r reads (r + 0.05) / 10
    sel = hit & (raw > 0.3) & (raw < 5.0)  # std = 1e-5 (r^2 + r + 1) <= 0.31 mm there
    assert np.allclose(px.cpu().numpy()[sel], (raw[sel] + 0.05) / 10.0, atol=2e-4)
