"""The reference's RL front-ends against this package (SURVEY 8b: "must drop in unchanged"), on the CPU twins:

  * rl_training/rl_games/runner.py       -- the module is executed as it is (rl_games itself is not installed: its two registries
                                             `env_configurations` / `vecenv` are stubbed by dicts, `gym` by a 20-line Wrapper / Box);
                                             every env it registers (except the two articulated-robot tasks) is built through ITS
                                             AERIALRLGPUEnv + ExtractObsWrapper and stepped;
  * rl_training/cleanrl/ppo_continuous_action.py -- the whole script, __main__ included: two PPO updates on position_setpoint_task;
  * rl_training/sample_factory/.../train_aerialgym.py -- its AerialGymVecEnv class (lifted out by name; sample_factory is not
                                             installed), reset / step through it.
Needs a reference checkout named by AERIAL_GYM_REFERENCE: skipped elsewhere."""
import ast
import os
import sys
import types

import numpy as np
import pytest
import torch

RL = os.path.join(os.environ.get("AERIAL_GYM_REFERENCE", ""), "aerial_gym/rl_training")
pytestmark = pytest.mark.skipif(not os.path.isdir(RL), reason="reference checkout not present")

from ._cpu_stack import cpu_stack  # noqa: E402


class _Wrapper:  # gym.Wrapper as far as the reference's wrappers rely on it
    def __init__(self, env):
        self.env = env

    def __getattr__(self, name):
        return getattr(self.env, name)

    def reset(self, **kw):
        return self.env.reset(**kw)

    def step(self, action):
        return self.env.step(action)


class _Box:
    def __init__(self, low, high, shape=None, dtype=np.float32):
        self.low, self.high = np.asarray(low), np.asarray(high)
        self.shape = self.low.shape if shape is None else shape


@pytest.fixture
def stack(monkeypatch, tmp_path):
    import aerial_gym_simulator_b200.compat as compat
    import aerial_gym_simulator_b200.task  # noqa: F401
    from aerial_gym_simulator_b200.registry._core import task_registry
    from aerial_gym_simulator_b200.utils import helpers
    compat.install()
    if not hasattr(np, "Inf"):
        monkeypatch.setattr(np, "Inf", np.inf, raising=False)  # runner.py:74 predates numpy 2
    gym = types.ModuleType("gym")
    gym.Wrapper, gym.Env = _Wrapper, object
    gym.spaces = types.ModuleType("gym.spaces")
    gym.spaces.Box, gym.spaces.Dict = _Box, dict
    for name, mod in (("gym", gym), ("gym.spaces", gym.spaces), ("gymnasium", gym), ("gymnasium.spaces", gym.spaces)):
        monkeypatch.setitem(sys.modules, name, mod)
    for cfg in task_registry.get_task_configs():
        if isinstance(getattr(cfg, "device", None), str):
            monkeypatch.setattr(cfg, "device", "cpu")
    real_parse = helpers.parse_arguments

    def parse_on_cpu(*a, **k):  # "--sim_device cpu" is refused by the product (no CPU pipeline); the twin stands in for the GPU here
        args = real_parse(*a, **k)
        args.sim_device_type = "cpu"
        return args
    monkeypatch.setattr(helpers, "parse_arguments", parse_on_cpu)
    monkeypatch.setattr(sys.modules["aerial_gym.utils.helpers"], "parse_arguments", parse_on_cpu, raising=False)
    monkeypatch.chdir(tmp_path)
    with cpu_stack() as proxy:
        yield proxy


def test_rl_games_runner_module(stack, monkeypatch):
    configurations, vec_types = {}, {}
    envc = types.ModuleType("rl_games.common.env_configurations")
    envc.configurations, envc.register = configurations, lambda name, cfg: configurations.__setitem__(name, cfg)
    vecenv = types.ModuleType("rl_games.common.vecenv")
    vecenv.IVecEnv, vecenv.register = object, lambda name, fn: vec_types.__setitem__(name, fn)
    common = types.ModuleType("rl_games.common")
    common.env_configurations, common.vecenv = envc, vecenv
    for name, mod in (("rl_games", types.ModuleType("rl_games")), ("rl_games.common", common),
                      ("rl_games.common.env_configurations", envc), ("rl_games.common.vecenv", vecenv)):
        monkeypatch.setitem(sys.modules, name, mod)
    if "distutils" not in sys.modules:
        try:
            import distutils  # noqa: F401
        except ImportError:
            monkeypatch.setitem(sys.modules, "distutils", types.ModuleType("distutils"))
    path = os.path.join(RL, "rl_games", "runner.py")
    g = {"__name__": "reference_runner", "__file__": path}
    exec(compile(open(path).read(), path, "exec"), g)
    assert set(vec_types) == {"AERIAL-RLGPU"}
    articulated = {"position_setpoint_task_reconfigurable", "position_setpoint_task_morphy"}
    assert articulated < set(configurations) and len(configurations) == 9
    expect = {"position_setpoint_task": (13, 4), "navigation_task": (81, 4), "lidar_navigation_task": (337, 4)}
    for name in sorted(set(configurations) - articulated):
        env = vec_types["AERIAL-RLGPU"](name, 1, num_envs=6, headless=True, seed=2, use_warp=True)
        info = env.get_env_info()
        D, A = info["observation_space"].shape[0], info["action_space"].shape[0]
        if name in expect:
            assert (D, A) == expect[name]
        obs = env.reset()
        assert torch.is_tensor(obs) and obs.shape == (6, D)
        for _ in range(3):
            obs, rew, dones, infos = env.step(torch.zeros(6, A))
        assert obs.shape == (6, D) and rew.shape == (6,) and dones.shape == (6,) and isinstance(infos, dict)
        assert torch.isfinite(obs).all() and torch.isfinite(rew).all()
        env.env.env.close()
    # its argument parsing (gymutil / parse_arguments with the trainer's own parameter table) and config update
    monkeypatch.setattr(sys, "argv", ["runner.py", "--task", "position_setpoint_task", "--num_envs", "512", "--headless", "True", "--train"])
    args = vars(g["get_args"]())
    assert args["task"] == "position_setpoint_task" and args["num_envs"] == 512 and args["headless"] is True and args["train"]
    cfg = g["update_config"]({"params": {"seed": 1, "config": {"env_config": {}}}}, args)
    assert cfg["params"]["config"]["env_config"] == {"headless": True, "num_envs": 512, "use_warp": True} and cfg["params"]["config"]["num_actors"] == 512


def test_cleanrl_ppo_script_runs_two_updates(stack, monkeypatch, capsys):
    path = os.path.join(RL, "cleanrl", "ppo_continuous_action.py")
    from aerial_gym_simulator_b200.config.task_config import position_setpoint_task_config as C
    monkeypatch.setattr(C, "num_envs", 32)
    monkeypatch.setattr(sys, "argv", ["ppo_continuous_action.py", "--task", "position_setpoint_task", "--num_envs", "32", "--num-steps", "8",
                                      "--total-timesteps", "512", "--update-epochs", "1", "--num-minibatches", "2", "--seed", "3"])
    g = {"__name__": "__main__", "__file__": path}
    exec(compile(open(path).read(), path, "exec"), g)
    out = capsys.readouterr().out
    assert "num actions:  4" in out and "num obs:  13" in out and out.count("SPS:") == 2
    assert g["global_step"] == 512 and torch.isfinite(g["v_loss"]) and torch.isfinite(g["pg_loss"])
    assert int(g["envs"].episode_lengths.max()) <= 16


def test_sample_factory_vec_env_class(stack):
    path = os.path.join(RL, "sample_factory", "aerialgym_examples", "train_aerialgym.py")
    tree = ast.parse(open(path).read())
    cls = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "AerialGymVecEnv")
    import gymnasium as gym
    from typing import Dict, Tuple
    from aerial_gym.registry.task_registry import task_registry
    g = {"gym": gym, "torch": torch, "Tensor": torch.Tensor, "Dict": Dict, "Tuple": Tuple, "convert_space": lambda s: s}
    exec(compile(ast.Module([cls], []), path, "exec"), g)
    env = g["AerialGymVecEnv"](task_registry.make_task(task_name="position_setpoint_task", num_envs=5, headless=True), "obs")
    assert env.num_agents == 5 and "observations" in env.observation_space and env.action_space.shape == (4,)
    obs, infos = env.reset()
    obs, rew, term, trunc, infos = env.step(torch.zeros(5, 4))
    assert obs["observations"].shape == (5, 13) and term.dtype == trunc.dtype == torch.bool
