"""Env-sharded tasks through the product API (task_registry.make_task(..., args={"world_size": W, "rank": r})): the observation handed to the
policy is the all-gathered [W * N, D] tensor (SURVEY 8e).  On one GPU the world is emulated (args["loopback"]): the protocol -- ring, push /
gate / wait kernels, flag words -- runs for real, the peers' rows stay zero.  With >= 2 GPUs tools/check_sharded_task.py runs it under torchrun
against NCCL's all_gather."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _make(name, n, args, seed=5):
    import aerial_gym_simulator_b200.task  # noqa: F401
    from aerial_gym_simulator_b200.registry.task_registry import task_registry

    cfg = task_registry.get_task_config(name)
    old = (getattr(cfg, "args", None), cfg.device)
    cfg.device, cfg.args = DEV, None
    try:
        return task_registry.make_task(name, seed=seed, num_envs=n, headless=True, args=args)
    finally:
        cfg.args, cfg.device = old


def test_sharded_position_task_loopback_equals_unsharded():
    n = 4096
    plain = _make("position_setpoint_task", n, None)
    shard = _make("position_setpoint_task", n, {"world_size": 2, "rank": 0, "loopback": True})
    assert shard.obs_gather is not None and shard.shard_world == 2 and plain.obs_gather is None
    o_p, o_s = plain.reset()[0], shard.reset()[0]
    assert o_s["observations"].shape == (2 * n, 13) and o_s["observations_local"].shape == (n, 13)
    torch.cuda.synchronize()
    assert torch.equal(o_s["observations_local"], o_p["observations"]) and torch.equal(o_s["observations"][:n], o_p["observations"])
    g = torch.Generator(device=DEV).manual_seed(2)
    for step in range(25):
        a = torch.rand(n, 4, generator=g, device=DEV) * 2 - 1
        (op, rp, tp, up, _), (os_, rs, ts, us, _) = plain.step(a), shard.step(a)
        torch.cuda.synchronize()
        assert torch.equal(os_["observations_local"], op["observations"]), f"step {step}"
        assert torch.equal(os_["observations"][:n], op["observations"]) and not os_["observations"][n:].any()
        assert torch.equal(rs, rp) and torch.equal(ts, tp) and torch.equal(us, up)
    shard.obs_gather.check()
    shard.sim_env.engine.check()
    shard.close()
    plain.close()


def test_sharded_navigation_task_loopback():
    n = 16
    shard = _make("navigation_task", n, {"world_size": 3, "rank": 0, "loopback": True}, seed=7)
    D = shard.task_config.observation_space_dim
    obs = shard.reset()[0]
    assert obs["observations"].shape == (3 * n, D) and obs["observations_local"].shape == (n, D)
    a = torch.zeros(n, shard.task_config.action_space_dim, device=DEV)
    for _ in range(3):
        obs = shard.step(a)[0]
        torch.cuda.synchronize()
        assert torch.equal(obs["observations"][:n], obs["observations_local"]) and not obs["observations"][n:].any()
        assert torch.isfinite(obs["observations"]).all() and obs["observations_local"].abs().sum() > 0
    shard.obs_gather.check()
    shard.close()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_sharded_position_task_two_ranks_equals_nccl():
    env = dict(os.environ, NCCL_DEBUG="WARN")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                        "--master-port", "29541", os.path.join(ROOT, "tools", "check_sharded_task.py")], capture_output=True, text=True, env=env, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    line = [l for l in r.stdout.splitlines() if l.startswith("SHARDED_TASK")][-1]
    assert "global_obs_equals_nccl=True" in line and "local_rows_in_place=True" in line, line
