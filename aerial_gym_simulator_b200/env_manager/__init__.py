"""EnvManager: the orchestrator surface of the reference (env_manager/env_manager.py) over the
H100 engines.  Registers the env / sim configs (env_manager/__init__.py, sim/__init__.py)."""
from ..config import env_config as _ec
from ..config import sim_config as _sc
from ..registry._core import env_config_registry, sim_config_registry

env_config_registry.register("empty_env", _ec.EmptyEnvCfg)
env_config_registry.register("env_with_obstacles", _ec.EnvWithObstaclesCfg)
env_config_registry.register("env_with_lidar_nav_obstacles", _ec.EnvWithLidarNavObstaclesCfg)
env_config_registry.register("dynamic_env", _ec.DynamicEnvironmentCfg)
env_config_registry.register("empty_env_2ms", _ec.EnvCfg2Ms)
env_config_registry.register("forest_env", _ec.ForestEnvCfg)
sim_config_registry.register("base_sim", _sc.BaseSimConfig)
sim_config_registry.register("base_sim_headless", _sc.BaseSimHeadlessConfig)
sim_config_registry.register("base_sim_2ms", _sc.SimCfg2Ms)
sim_config_registry.register("base_sim_4ms", _sc.SimCfg4Ms)
sim_config_registry.register("custom_sim", _sc.CustomSimConfig)

from ..config.env_config import (DynamicEnvironmentCfg, EmptyEnvCfg, EnvCfg2Ms, EnvWithLidarNavObstaclesCfg,  # noqa: E402,F401
                                 EnvWithObstaclesCfg, ForestEnvCfg)
from .env_manager import EnvManager  # noqa: E402,F401
