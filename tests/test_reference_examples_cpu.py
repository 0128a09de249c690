"""The reference's own example scripts, UNMODIFIED in what they import and call, run against this package through
compat.install() on the CPU twins (tests/_cpu_stack.py).  Only three textual substitutions are made before exec:
"cuda:0" -> "cpu" (no GPU here), the loop counts (10,000 steps -> a few dozen) and nothing else.  What this pins: every attribute
path, registry name, keyword and call the scripts use exists with the reference's meaning (SURVEY 8b "who calls").
Needs a reference checkout named by AERIAL_GYM_REFERENCE: skipped elsewhere."""
import os
import re
import sys

import pytest
import torch

EX = os.path.join(os.environ.get("AERIAL_GYM_REFERENCE", ""), "aerial_gym/examples")
pytestmark = pytest.mark.skipif(not os.path.isdir(EX), reason="reference checkout not present")

from ._cpu_stack import cpu_stack  # noqa: E402


def _run(script, steps, argv=(), subst=()):
    import aerial_gym_simulator_b200.compat as compat
    from aerial_gym_simulator_b200.registry._core import task_registry
    compat.install()
    src = open(os.path.join(EX, script)).read()
    src = src.replace('"cuda:0"', '"cpu"')
    for a, b in subst:
        assert a in src
        src = src.replace(a, b)
    if steps is not None:
        src, n = re.subn(r"range\((?:\d+|int\([^\n]*\))\):", f"range({steps}):", src)
        assert n >= 1, "no step loop found"
    saved_argv, saved_dev = sys.argv, {}
    import aerial_gym_simulator_b200.task  # noqa: F401
    for cfg in task_registry.get_task_configs():
        if isinstance(getattr(cfg, "device", None), str):
            saved_dev[cfg] = cfg.device
            cfg.device = "cpu"
    sys.argv = [script, *argv]
    g = {"__name__": "__main__", "__file__": os.path.join(EX, script)}
    try:
        with cpu_stack() as proxy:
            exec(compile(src, script, "exec"), g)
    finally:
        sys.argv = saved_argv
        for cfg, d in saved_dev.items():
            cfg.device = d
    return g, proxy


def test_position_control_example():
    g, _ = _run("position_control_example.py", 40, ["--num_envs", "8", "--headless", "True"])
    env = g["env_manager"]
    assert env.num_envs == 8 and torch.isfinite(env.global_tensor_dict["robot_state_tensor"]).all()


def test_acceleration_control_example():
    g, _ = _run("acceleration_control_example.py", 12)
    env = g["env_manager"]
    assert env.num_envs == 16 and env.sensor is None  # base_quadrotor carries no camera
    assert torch.isfinite(env.global_tensor_dict["robot_state_tensor"]).all()


def test_benchmark_example():
    g, _ = _run("benchmark.py", 120)
    assert g["env_manager"].num_envs == 256 and g["elapsed_steps"] == 20


def test_dynamic_env_example():
    g, proxy = _run("dynamic_env_example.py", 6, ["--num_envs", "4", "--headless", "True", "--use_warp", "True"])
    assert g["num_assets_in_env"] == g["env_manager"].IGE_env.num_assets_per_env - 1 and proxy.calls["agx_obstacle_step"] == 6


def test_rl_env_example():
    g, _ = _run("rl_env_example.py", 8)
    assert g["obs"]["observations"].shape[1] == 13 and g["reward"].shape == g["terminated"].shape == g["truncated"].shape


def test_navigation_task_example():
    g, _ = _run("navigation_task_example.py", 3)
    assert g["obs"]["observations"].shape == (16, 81)


def test_imu_data_collection_example():
    g, proxy = _run("imu_data_collection.py", 5)
    assert g["imu_measurement"].shape == (6,) and g["sim_dt"] == g["env_manager"].sim_config.sim.dt


def test_position_control_example_rov():
    # the script names a controller the reference does not register either (control/__init__.py:99 registers
    # "rov_fully_actuated_control"): same ValueError from the registry here as there
    with pytest.raises(ValueError, match="fully_actuated_control"):
        _run("position_control_example_rov.py", 20)
    g, _ = _run("position_control_example_rov.py", 20, subst=[('"fully_actuated_control"', '"rov_fully_actuated_control"')])
    assert g["actions"].shape == (64, 7) and torch.isfinite(g["env_manager"].global_tensor_dict["robot_state_tensor"]).all()


@pytest.fixture
def fake_matplotlib(monkeypatch):
    """matplotlib is not installed: the camera scripts only use cm.plasma(x) -> RGBA in [0, 1]"""
    import types

    import numpy as np
    mpl, cm, image = types.ModuleType("matplotlib"), types.ModuleType("matplotlib.cm"), types.ModuleType("matplotlib.image")
    cm.plasma = lambda x: np.stack([x, 1.0 - x, 0.5 * np.ones_like(x), np.ones_like(x)], axis=-1)
    mpl.cm, mpl.image = cm, image
    for name, mod in (("matplotlib", mpl), ("matplotlib.cm", cm), ("matplotlib.image", image)):
        monkeypatch.setitem(sys.modules, name, mod)


def test_save_camera_stream_example(fake_matplotlib, tmp_path, monkeypatch):
    """stereo depth camera + segmentation in env_with_obstacles; 2 frames (the gif-saving branch needs 100)"""
    monkeypatch.chdir(tmp_path)
    g, _ = _run("save_camera_stream.py", 2)
    env = g["env_manager"]
    assert env.sensor is not None and "stereo" in env.robot_manager.robot.cfg.sensor_config.camera_config.__name__.lower()
    assert len(g["depth_frames"]) == 2 and g["depth_frames"][0].size == (g["image1"].shape[1], g["image1"].shape[0])
    assert g["seg_image1_normalized"].min() == 0.0 and g["seg_image1_normalized"].max() == 1.0


def test_save_camera_stream_normal_faceID_example(fake_matplotlib, tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    g, _ = _run("save_camera_stream_normal_faceID.py", 2)
    assert g["env_manager"].sensor is not None and len(g["merged_image_frames"]) == 2


def test_user_subclass_of_navigation_task():
    """examples/dce_rl_navigation/dce_navigation_task.py: a USER subclass of NavigationTask that overrides process_obs_for_task and reads
    the parent's attributes (obs_dict, task_obs, target_position, image_latents) -- the class-level contract, not only the call surface"""
    import aerial_gym_simulator_b200.compat as compat
    compat.install()
    from aerial_gym_simulator_b200.config.task_config import navigation_task_config
    path = os.path.join(EX, "dce_rl_navigation", "dce_navigation_task.py")
    g = {"__name__": "dce_navigation_task", "__file__": path}
    exec(compile(open(path).read(), path, "exec"), g)
    cfg = type("cfg", (navigation_task_config,), {"curriculum": type("curriculum", (navigation_task_config.curriculum,), {})})
    cfg.device, cfg.num_envs = "cpu", 32
    with cpu_stack() as proxy:
        task = g["DCE_RL_Navigation_Task"](cfg, seed=1, headless=True)
        assert task.task_config.num_envs == 16 and task.task_config.action_space_dim == 3 and task.task_config.curriculum.min_level == 36
        task.reset()
        for _ in range(2):
            obs, rew, term, trunc, info = task.step(torch.zeros(16, 3))
    o = obs["observations"]
    assert o.shape == (16, 81) and torch.isfinite(o).all() and (o[:, 6] == 0).all()
    assert torch.allclose(o[:, 0:3].norm(dim=1), torch.ones(16), atol=1e-5)  # the subclass's own layout: unit vector, distance / 5
    assert torch.equal(o[:, 17:81], task.image_latents) and proxy.calls["agx_nav_reward"] == 2 and "agx_nav_obs" not in proxy.calls


def test_sys_id_example(monkeypatch, capsys):
    """examples/sys_id.py, all 4 x 500 steps of it (only "cuda:0" -> "cpu"; pyplot stubbed): a velocity step response of lmf2.  It reads
    the tensors of env_manager.get_obs() ONCE and relies on them being updated in place by every step; the printed time constants are
    the closed-loop response times of the three velocity axes and the yaw rate."""
    import types

    class _Any:
        def __getattr__(self, n):
            return _Any()

        def __call__(self, *a, **k):
            return _Any()

        def __getitem__(self, i):
            return _Any()
    plt = types.ModuleType("matplotlib.pyplot")
    plt.subplots = lambda *a, **k: (_Any(), _Any())
    plt.show = lambda *a, **k: None
    mpl = types.ModuleType("matplotlib")
    mpl.pyplot = plt
    monkeypatch.setitem(sys.modules, "matplotlib", mpl)
    monkeypatch.setitem(sys.modules, "matplotlib.pyplot", plt)
    g, _ = _run("sys_id.py", None, ["--num_envs", "4", "--headless", "True"])
    out = capsys.readouterr().out
    taus = [float(l.split(":")[1]) for l in out.splitlines() if l.startswith("Time Constant")]
    assert len(taus) == 4 and all(0.05 < t < 2.0 for t in taus), taus  # every axis reaches 63 % of the commanded step within 2 s
    seq = g["observation_sequence_np"]
    assert seq.shape == (500, 4, 4) and abs(seq[-1, 0, 3] - 1.0) < 0.2  # last run: yaw rate settles near the commanded 1 rad/s
