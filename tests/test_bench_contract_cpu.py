"""The bench line contract, checked on the committed lines H100 runs printed (`profiles/bench_h100_n*.json`) and on the reference
arm run on the host cores: the keys a consumer of the line reads, the roofline arithmetic, the multi-GPU self-check."""
import glob
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LINES = sorted(glob.glob(os.path.join(ROOT, "profiles", "bench_h100_n*.json")))
BASE_KEYS = {"metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline", "dtype",
             "data", "config", "roofline", "e2e", "gpu_launches", "clocks"}


def _load(path):
    with open(path) as f:
        return json.loads(f.read().strip().splitlines()[-1])


@pytest.mark.parametrize("path", LINES, ids=[os.path.basename(p) for p in LINES])
def test_committed_bench_lines_follow_the_contract(path):
    d = _load(path)
    assert BASE_KEYS <= set(d), BASE_KEYS - set(d)
    n = d["n_gpus"]
    assert d["unit"] == "env-steps/s" and d["higher_is_better"] is True and d["scaling"] == "weak" and d["data"] == "synthetic"
    assert d["dtype"] == "f32" and d["vs_baseline"] is None  # BASELINE.md has no published number for this metric
    assert d["warmup"] >= 3 and d["gpu_launches"] >= d["steps"]
    cfg = d["config"]
    assert cfg["envs_per_gpu"] == 65536 and cfg["global_envs"] == 65536 * n and "workload" in cfg and "model" not in cfg
    # value = whole-job units / device time of the timed region
    assert d["value"] == pytest.approx(cfg["global_envs"] / (d["ms_per_step"] * 1e-3), rel=1e-6)
    r = d["roofline"]
    assert r["bound"] == "hbm" and r["unit"] == "GB/s" and r["frac"] == pytest.approx(r["achieved"] / r["peak"], rel=1e-9)
    assert r["algorithmic_bytes_per_launch"] == 210 * 65536  # DESIGN section 6: 210 B per env-step
    assert r["achieved"] == pytest.approx(r["algorithmic_bytes_per_launch"] / (r["kernel_ms_avg"] * 1e-3) / 1e9, rel=1e-6)
    e = d["e2e"]
    assert e["value"] > 0 and e["h2d_bytes_per_step"] > 0 and e["d2h_bytes_per_step"] > 0 and e["value"] < d["value"]
    c = d["clocks"]
    assert c["sm_mhz"] > 0.9 * c["sm_max_mhz"] and not set(c["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}
    if n == 1:
        b = d["cpu_baseline"]
        # "port" = the oracle port of the same step, timed where the reference checkout was not staged (bench.py time_cpu_reference)
        assert b["kind"] in ("reference", "port") and b["cores"] >= 1 and b["value"] > 0 and "sample" in b
        for sub in ("hp2_depth", "config3_depth_270x480_1024box", "config4_lidar_64x512_octarotor", "config5_env_sweep",
                    "navigation_task_e2e"):
            assert sub in d, sub
        assert r["nvlink_floor_us"] is None
    else:
        # the hand-written gather is checked against NCCL inside the same run, and the wire floor is printed next to the step
        assert d["obs_gather_check"] is True
        assert r["nvlink_floor_us"] == pytest.approx((n - 1) * 65536 * 52 / 450e9 * 1e6, rel=1e-3)
        assert d["ms_per_step"] * 1e3 > r["nvlink_floor_us"]  # nobody beats the wire
        assert d["value_obs_gather_sync"] < d["value"]


def test_reference_arm_line_here():
    """`bench.py --impl reference` on this host: same metric / config keys, impl + cpu_baseline + zero-byte e2e, one JSON line on stdout."""
    from oracle import reference_arm
    if not reference_arm.staged():
        pytest.skip("baseline/_ref is not staged (__graft_entry__.build() stages it where AERIAL_GYM_REFERENCE names a reference checkout)")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "1", "--steps", "2", "--warmup", "1",
                        "--envs", "4096"], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    out = [l for l in r.stdout.splitlines() if l.strip()]
    assert len(out) == 1, out
    d = json.loads(out[0])
    assert d["impl"] == "reference" and d["unit"] == "env-steps/s" and d["higher_is_better"] is True
    assert d["cpu_baseline"]["kind"] == "reference" and d["cpu_baseline"]["value"] == d["value"]
    assert d["e2e"] == {"value": d["value"], "unit": d["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
