"""Timing of the small kernels around the two hot paths (not part of bench.py's contract line):

    python tools/bench_aux.py [--envs 4096] [--iters 200]          # one JSON line per kernel on stdout

Each kernel is timed with CUDA events on torch's current stream after 10 warm-up launches, inputs rotated over enough replicas to
exceed the H100's 50 MB L2; `achieved` = algorithmic bytes (DESIGN 6, "Kernels written after the GPU budget was spent") / mean launch time,
`frac` against MEASURED_PEAKS.json's HBM figure (fallback 3350 GB/s, the H100 SXM data sheet)."""
import argparse
import ctypes as C
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from aerial_gym_simulator_b200 import _lib  # noqa: E402


def peak_gbs():
    try:
        d = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
        for k in ("hbm_gbs", "hbm_gbs_burst", "hbm_copy_gbs"):
            if k in d:
                return float(d[k]), f"MEASURED_PEAKS.json {k}"
    except Exception:  # noqa: BLE001
        pass
    return 3350.0, "H100 SXM data sheet (fallback)"


def timeit(fn, reps, iters):
    for i in range(10):
        fn(i % reps)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(iters):
        fn(i % reps)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e-3


def p(t):
    return C.c_void_p(t.data_ptr())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--iters", type=int, default=200)
    a = ap.parse_args()
    dev, lib, N = "cuda:0", _lib.load(), a.envs
    peak, src = peak_gbs()
    out = []

    def report(name, bytes_per_launch, t, units, unit_name):
        out.append({"kernel": name, "ms": t * 1e3, "algorithmic_bytes": bytes_per_launch, "achieved_gbs": bytes_per_launch / t / 1e9,
                    "peak_gbs": peak, "frac": bytes_per_launch / t / 1e9 / peak, "peak_source": src, unit_name + "_per_s": units / t, "envs": N})
        print(json.dumps(out[-1]))

    # ---- agx_lidar_nav_pool: 48 x 120 x 12 B in, 16 x 20 x 4 + 4 B out per env
    H, W = 48, 120
    per_env = H * W * 12 + 52 + (H // 3) * (W // 6) * 4 + 4
    reps = max(2, int(200e6 // (N * per_env)) + 1)
    pcs = [torch.randn(N, H, W, 3, device=dev) * 5 for _ in range(reps)]
    st = torch.randn(N, 13, device=dev)
    ds, ttc = torch.zeros(N, H // 3, W // 6, device=dev), torch.zeros(N, device=dev)
    t = timeit(lambda i: _lib.check(lib.agx_lidar_nav_pool(N, H, W, 3, 6, p(pcs[i]), p(st), 13, 10.0, 0.2, 10.0, 10.0, p(ds), p(ttc), None),
                                    "agx_lidar_nav_pool"), reps, a.iters)
    report("lidar_nav_pool_kernel", N * per_env, t, N, "envs")
    del pcs
    # ---- agx_hp2_noise_limits: 4 B in + 4 B out per value (270 x 480 depth image per env, capped at 64 M values)
    P = min(N * 270 * 480, 64 * 1024 * 1024)
    reps = max(2, int(200e6 // (P * 4)) + 1)
    imgs = [torch.rand(P, device=dev) * 12 for _ in range(reps)]
    n = _lib.AgxHp2Noise()
    n.components, n.enable_noise, n.apply_limits, n.normalize = 1, 1, 1, 1
    n.std_a, n.std_b, n.std_c, n.mean_offset, n.pixel_dropout_prob = 0.00038089, -0.00343351, 0.01553284, -0.025, 0.01
    n.max_range, n.min_range, n.far_out_of_range_value, n.near_out_of_range_value = 10.0, 0.2, 10.0, -10.0
    t = timeit(lambda i: _lib.check(lib.agx_hp2_noise_limits(p(imgs[i]), P, 0, C.byref(n), 1234, i, None), "agx_hp2_noise_limits"), reps, a.iters)
    report("noise_limits_kernel", P * 8, t, P, "values")
    del imgs
    # ---- agx_e2e_reward + agx_e2e_obs (launch-latency bound at the tasks' 4096 envs; reported for completeness)
    s13 = torch.randn(N, 13, device=dev)
    s13[:, 3:7] = torch.nn.functional.normalize(s13[:, 3:7], dim=1)
    w, act, prev, perr, noise = (torch.randn(N, k, device=dev) for k in (3, 4, 4, 3, 12))
    cr, rew, obs = torch.zeros(N, dtype=torch.uint8, device=dev), torch.zeros(N, device=dev), torch.zeros(N, 15, device=dev)
    prm = _lib.AgxE2ERewardParams()
    for k, v in dict(z_error_scale=11.0, align_gain1=6.0, align_exp1=5.0, angvel_gain=0.3, hover_thrust=0.912, towards_gain_pos=10.0,
                     towards_gain_neg=15.0, action_diff_gain=1.3, crash_dist=1.5).items():
        setattr(prm, k, v)
    t = timeit(lambda i: (_lib.check(lib.agx_e2e_reward(N, p(s13), 13, p(w), None, p(act), p(prev), p(perr), C.byref(prm), p(cr), p(rew), None), "r"),
                          _lib.check(lib.agx_e2e_obs(N, p(s13), 13, p(w), None, p(noise), p(obs), 15, None), "o")), 1, a.iters)
    report("e2e_reward_kernel + e2e_obs_kernel", N * (2 * (52 + 12) + 44 + 48 + 5 + 60), t, N, "envs")


if __name__ == "__main__":
    main()
