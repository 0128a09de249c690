"""PositionSetpointTask (task/position_setpoint_task/position_setpoint_task.py:20-282).

step() is ONE C-ABI call (agx_hp1_position_task_step): physics, sim_steps, reward + crash,
truncation, reset of finished envs and the 13-D observation are fused in the HP1 kernel; the
tensors returned are the same objects every call, mutated in place, like the reference.

task_config.args:
  {"reset_rng": "device"}  (default) in-kernel Philox resets -> single launch, no host sync;
  {"reset_rng": "torch"}   reference-order torch draws; the host reads the any-reset flag each
                           step exactly where the reference syncs (env_manager.py:364-375).
  {"host_io": True}        observations / rewards / terminations / truncations are pinned HOST tensors
                           the kernel writes directly (agx_host_alloc), `actions` may be a pinned host
                           tensor the kernel reads in place; step() returns after the stream has drained,
                           so the results can be read at once.  For consumers that live on the host."""
import numpy as np
import torch

from ..sim import SimBuilder
from .base_task import BaseTask
from .spaces import Box, Dict


class PositionSetpointTask(BaseTask):
    def __init__(self, task_config, seed=None, num_envs=None, headless=None, device=None, use_warp=None):
        for k, v in (("seed", seed), ("num_envs", num_envs), ("headless", headless), ("device", device), ("use_warp", use_warp)):
            if v is not None:
                setattr(task_config, k, v)
        super().__init__(task_config)
        self.device = self.task_config.device
        for key in list(self.task_config.reward_parameters.keys()):
            self.task_config.reward_parameters[key] = torch.as_tensor(self.task_config.reward_parameters[key], device=self.device)
        args = dict(self.task_config.args or {})
        args.setdefault("seed", self._seed)
        world, rank, _ = self.shard_spec()
        if world > 1:  # env-sharded: this rank's envs are the global ids rank * num_envs ... (keys the device RNG)
            args.setdefault("env_id_offset", rank * int(self.task_config.num_envs))
        self.sim_env = SimBuilder().build_env(
            sim_name=self.task_config.sim_name, env_name=self.task_config.env_name, robot_name=self.task_config.robot_name,
            controller_name=self.task_config.controller_name, args=args, device=self.device,
            num_envs=self.task_config.num_envs, use_warp=self.task_config.use_warp, headless=self.task_config.headless)
        env, eng = self.sim_env, self.sim_env.engine
        if env.spec.num_actions != self.task_config.action_space_dim:
            raise ValueError("task action_space_dim does not match the controller's action count")
        eng.cfg.episode_len_steps = int(self.task_config.episode_len_steps)
        self.num_envs = env.num_envs
        # a disturbance-enabled robot in an env with several (or a random number of) physics sub-steps per env step needs a fresh draw
        # per sub-step: the fused one-launch step cannot do that, the reference-order sequence over EnvManager.step can (decided
        # here, once, so that no step consumes random.gauss and then fails)
        e = env.cfg.env
        self._unfused = bool(env.spec.enable_disturbance and (e.num_physics_steps_per_env_step_mean != 1 or e.num_physics_steps_per_env_step_std != 0))
        # an articulated robot has no fused step: its physics is agx_hp1_articulated_step, the rest of the step the same sequence
        self._unfused = self._unfused or env.articulated
        self.actions = torch.zeros((self.num_envs, self.task_config.action_space_dim), device=self.device)
        self.prev_actions = torch.zeros_like(self.actions)
        self.counter = 0
        self._published_epoch = -1
        self.target_position = eng.target_position  # [N,3], read by the kernel
        self.obs_dict = env.get_obs()
        self.obs_dict["num_obstacles_in_env"] = 1
        self.terminations = self.obs_dict["crashes"]
        self.truncations = self.obs_dict["truncations"]
        self.rewards = eng.reward
        self.observation_space = Dict({"observations": Box(low=-1.0, high=1.0, shape=(13,), dtype=np.float32)})
        self.action_space = Box(low=-1.0, high=1.0, shape=(self.task_config.action_space_dim,), dtype=np.float32)
        self.task_obs = {
            "observations": eng.obs,
            "priviliged_obs": torch.zeros((self.num_envs, self.task_config.privileged_observation_space_dim), device=self.device),
            "collisions": torch.zeros((self.num_envs, 1), device=self.device),
            "rewards": self.rewards,
            "terminations": self.terminations,
            "truncations": self.truncations,
        }
        self.infos = {}
        if self.init_sharding(self.num_envs, 13, self.device) is not None:
            if eng.host_io:
                raise ValueError("args['host_io'] and a sharded task are mutually exclusive")
            eng.attach_obs_gather(self.obs_gather)  # the fused step writes its observation into the gather's ring; the push runs beside it

    def close(self):
        if getattr(self, "obs_gather", None) is not None and self.sim_env.engine is not None:
            self.sim_env.engine.attach_obs_gather(None)
        self.sim_env.delete_env()

    def reset(self):
        self.target_position[:, 0:3] = 0.0
        self.infos = {}
        self.sim_env.reset()
        if self._overridden("process_obs_for_task"):
            self.process_obs_for_task()
        return self.get_return_tuple()

    def reset_idx(self, env_ids):
        self.target_position[:, 0:3] = 0.0
        self.infos = {}
        self.sim_env.reset_idx(env_ids)

    def render(self):
        return None

    def step(self, actions):
        self.counter += 1
        env, eng = self.sim_env, self.sim_env.engine
        if actions.dtype != torch.float32 or not actions.is_contiguous():
            actions = actions.float().contiguous()
        if self._overridden("compute_rewards_and_crashes") or self.task_config.return_state_before_reset or self._unfused:
            return self._step_with_reward_hook(actions)  # (the fused step resets inside the launch: nothing to return "before")
        if eng.host_io and actions.device.type == "cpu" and not actions.is_pinned():
            eng.host_actions.copy_(actions)  # pageable host memory: stage through the mapped buffer
            actions = eng.host_actions
        self.prev_actions, self.actions = self.actions, actions  # the reference copies; nobody reads prev afterwards
        n = env.sample_physics_steps()  # consumes random.gauss like env_manager.py:417-425
        dist = env._draw_disturbance() if (env.spec.enable_disturbance and n == 1) else None  # (n != 1 with disturbances: _unfused)
        eng.position_task_step(actions, disturbance=dist, physics_steps=n)
        env.step_counter += 1
        if env.reset_rng == "torch":
            # reference flow: host decides, draws only when some env resets (env_manager.py:364-375)
            if int(eng.any_reset[0].item()) != 0:
                eng.any_reset.zero_()
                env.reset_idx(eng.reset_mask.nonzero(as_tuple=False).squeeze(-1))  # ends with the all-env refresh + obs
        env.render(render_components="sensors")
        if eng.host_io:
            torch.cuda.current_stream(eng.device).synchronize()  # results are in host memory now
        self.infos = {}
        if self._overridden("process_obs_for_task"):
            self.process_obs_for_task()
        return self.get_return_tuple()

    def get_return_tuple(self):
        if self.obs_gather is not None:
            self._publish_global_observations()
        return (self.task_obs, self.rewards, self.terminations, self.truncations, self.infos)

    def _publish_global_observations(self):
        """sharded task: task_obs['observations'] <- the gathered [W*N, 13] tensor of this step (waits for every rank's rows)"""
        g, eng = self.obs_gather, self.sim_env.engine
        if eng.gathered_obs is None or self._published_epoch == g.epoch:  # reset() / a hook path: the engine's observation was written outside the fused step
            glob, loc = self.gather_observations(eng.obs)
        else:
            if getattr(g, "peer_outs", None) is not None:
                g.loopback_complete(g.epoch)
            glob, loc = g.wait(), eng.obs
        self._published_epoch = g.epoch
        self.task_obs["observations"], self.task_obs["observations_local"] = glob, loc

    # ------------------------------------------------------------------------------------------
    # The reference's two hooks (position_setpoint_task.py:194-229).  For THIS class they are fused into the step kernel and never
    # called.  A subclass that overrides one gets the reference's behaviour:
    #   * only process_obs_for_task overridden: the fused step runs (reward, crash, truncation, reset, default observation in one
    #     launch), then the override rewrites task_obs -- same point in the sequence as get_return_tuple's call in the reference;
    #   * compute_rewards_and_crashes overridden: the step runs in the reference's order with the same kernels un-fused
    #     (physics launch -> the override -> truncation -> reset of finished envs -> observation hook).
    # The bodies below are what an override reaches through super(): plain torch on the env's device tensors.
    # ------------------------------------------------------------------------------------------
    def _overridden(self, name):
        return getattr(type(self), name) is not getattr(PositionSetpointTask, name)

    def process_obs_for_task(self):
        od, o = self.obs_dict, self.task_obs["observations"]
        o[:, 0:3] = self.target_position - od["robot_position"]
        o[:, 3:7] = od["robot_orientation"]
        o[:, 7:10] = od["robot_body_linvel"]
        o[:, 10:13] = od["robot_body_angvel"]
        self.task_obs["rewards"], self.task_obs["terminations"], self.task_obs["truncations"] = self.rewards, self.terminations, self.truncations

    def compute_rewards_and_crashes(self, obs_dict):
        """(reward [N], crashes [N] bool) of compute_reward (:245-282); writes the distance crashes into obs_dict["crashes"] like it"""
        q, crashes = obs_dict["robot_orientation"], obs_dict["crashes"]
        # the norm is rotation invariant, so the vehicle-frame rotation of the position error (:219-221) drops out
        dist = torch.norm(self.target_position - obs_dict["robot_position"], dim=1)
        pos_reward = 3.0 * torch.exp(-8.0 * dist * dist) + 2.0 * torch.exp(-4.0 * dist * dist)
        up_z = 1.0 - 2.0 * (q[:, 0] * q[:, 0] + q[:, 1] * q[:, 1])  # z component of the body z axis
        tilt = torch.abs(1.0 - up_z)
        spin = torch.norm(obs_dict["robot_body_angvel"], dim=1)
        reward = pos_reward + (20.0 - dist) / 40.0 + pos_reward * (0.2 / (0.1 + tilt * tilt) + 3.0 / (1.0 + spin * spin))
        crashes |= dist > 8.0
        return torch.where(crashes, torch.full_like(reward, -20.0), reward), crashes

    def _step_with_reward_hook(self, actions):
        env, cfg = self.sim_env, self.task_config
        if env.engine.host_io:
            raise NotImplementedError("args['host_io'] is a feature of the fused step; a reward override runs the un-fused sequence")
        self.prev_actions, self.actions = self.actions, actions
        env.step(actions=actions)                                                     # :163
        rew, crashes = self.compute_rewards_and_crashes(self.obs_dict)                # :168
        self.rewards[:], self.terminations[:] = rew, crashes
        before = self._hook_return_tuple() if cfg.return_state_before_reset else None  # :170-171
        self.truncations[:] = env.sim_steps > cfg.episode_len_steps                   # :172-174
        kept = self.task_obs["observations"].clone() if before is not None else None
        env.post_reward_calculation_step()                                            # :175
        self.infos = {}
        if before is None:
            return self._hook_return_tuple()
        self.task_obs["observations"].copy_(kept)  # (the engine's refresh after a reset rewrites its observation buffer)
        return before

    def _hook_return_tuple(self):
        self.process_obs_for_task()
        return (self.task_obs, self.rewards, self.terminations, self.truncations, self.infos)
