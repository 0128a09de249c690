"""Reference arm of bench.py: the reference's OWN control stack, unmodified, timed on the host cores.

TEST / MEASUREMENT INFRASTRUCTURE -- never imported by the product.  bench.py's `--impl reference` leg and `cpu_baseline` leg are
the only callers (and tests/test_reference_arm.py, which pins it against the oracle port).

What runs, per env step of position_setpoint_task (task/position_setpoint_task/position_setpoint_task.py:152-182 over
env_manager/env_manager.py:399-432), on torch CPU tensors:

  * `BaseMultirotor.step(actions)` (robots/base_multirotor.py:296-307) -- the reference's own update_states, Lee attitude
    controller, control allocation, motor model, drag and link force / torque tensors, imported UNMODIFIED from the copy of the
    reference that `__graft_entry__.build()` installs into `baseline/_ref` with
    `pip install --no-index --no-build-isolation --no-deps --target baseline/_ref` (stage(); the wheel's find_packages() skips the
    implicit namespace packages -- `aerial_gym/config`, `aerial_gym/registry`, `aerial_gym/task/<name>`, ... have no __init__.py
    but `aerial_gym.control` imports the first two at import time -- so stage() completes the install by copying the .py files
    the wheel missed next to the installed ones, byte for byte).  isaacgym and pytorch3d are closed / absent: empty `isaacgym.*` modules and the pytorch3d stub of
    tests/golden/_ref_loader.py stand in (the attitude controller calls neither).
  * the rigid-body integration that PhysX (`gym.simulate`, IGE_env_manager.py:477) performs in the reference is NOT available
    (closed binary): `oracle.hp1_oracle.link_wrenches_to_body` + `rigid_body_integrate` (our written spec) stand in;
  * the reference's `compute_reward` (position_setpoint_task.py:245-282), lifted out of its file with `ast` (the module itself
    imports isaacgym / gym), truncation, `BaseMultirotor.reset_idx` + the env-bounds draws of IGE_env_manager.py:513-519, and the
    13-D observation of process_obs_for_task (:194-203).

So `kind` = "reference": every line of the control stack is the reference's; the PhysX step is the one stand-in, and it is labelled."""
import ast
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
from tests.golden._ref_loader import REF_ROOT as REF_SRC  # noqa: E402  (AERIAL_GYM_REFERENCE: a checkout of the reference)
REF_DST = os.path.join(ROOT, "baseline", "_ref")


def staged() -> bool:
    return os.path.isdir(os.path.join(REF_DST, "aerial_gym", "control")) and os.path.isdir(os.path.join(REF_DST, "aerial_gym", "registry"))


def stage(force=False) -> str:
    """Install the unmodified reference into baseline/_ref (git-ignored, travels to the GPU box).  Needs a reference checkout (AERIAL_GYM_REFERENCE)."""
    if staged() and not force:
        return REF_DST
    if not os.path.isdir(os.path.join(REF_SRC, "aerial_gym")):
        raise RuntimeError("AERIAL_GYM_REFERENCE does not name a checkout of the reference: the reference arm cannot be staged")
    shutil.rmtree(REF_DST, ignore_errors=True)
    os.makedirs(REF_DST, exist_ok=True)
    with tempfile.TemporaryDirectory() as tmp:  # the reference checkout may be read-only and the build writes into the source tree
        src = os.path.join(tmp, "ref")
        shutil.copytree(REF_SRC, src, ignore=shutil.ignore_patterns(".git", "resources", "docs", "*.pth", "*.pt", "*.zip", "*.gif", "*.png"))
        r = subprocess.run([sys.executable, "-m", "pip", "install", "--no-index", "--no-build-isolation", "--no-deps", "--find-links",
                            "/opt/wheelhouse", "--target", REF_DST, src], capture_output=True, text=True)
        if r.returncode:
            raise RuntimeError("pip install of the reference failed:\n" + r.stdout[-2000:] + r.stderr[-2000:])
    # complete the install: every .py of the implicit namespace packages find_packages() does not see (config/, registry/,
    # task/<name>/, sensors/..., no __init__.py), byte for byte, next to the installed ones
    base = os.path.join(REF_SRC, "aerial_gym")
    for dirpath, dirnames, filenames in os.walk(base):
        dirnames[:] = [d for d in dirnames if d not in ("__pycache__", "resources")]
        for fn in filenames:
            if not fn.endswith(".py"):
                continue
            rel = os.path.relpath(os.path.join(dirpath, fn), base)
            dst = os.path.join(REF_DST, "aerial_gym", rel)
            if not os.path.exists(dst):
                os.makedirs(os.path.dirname(dst), exist_ok=True)
                shutil.copyfile(os.path.join(dirpath, fn), dst)
    return REF_DST


def _install_import_hooks():
    from tests.golden import _ref_loader

    root = REF_DST if staged() else REF_SRC
    if not os.path.isdir(os.path.join(root, "aerial_gym", "control")):
        raise RuntimeError("reference not staged: run __graft_entry__.build() in the build container (baseline/_ref)")
    _ref_loader.REF_ROOT = root
    _ref_loader.install()
    return root


def _reference_compute_reward(root):
    import torch
    from aerial_gym.utils import math as ref_math

    path = os.path.join(root, "aerial_gym", "task", "position_setpoint_task", "position_setpoint_task.py")
    tree = ast.parse(open(path).read())
    ns = {"torch": torch, "quat_axis": ref_math.quat_axis}
    for node in tree.body:
        if isinstance(node, ast.FunctionDef) and node.name in {"exp_func", "exp_penalty_func", "compute_reward"}:
            node.decorator_list = []  # @torch.jit.script removed: same arithmetic, eager (TorchScript cannot see the ast-loaded source)
            exec(compile(ast.Module(body=[node], type_ignores=[]), path, "exec"), ns)
    return ns["compute_reward"]


class ReferencePositionTask:
    """position_setpoint_task / base_quadrotor / lee_attitude_control / empty_env on the reference's own torch code (CPU)."""

    def __init__(self, num_envs, seed=0, episode_len_steps=500):
        import numpy as np
        import torch

        root = _install_import_hooks()
        import aerial_gym.control  # noqa: F401  (registers the reference's controllers)
        import aerial_gym.robots  # noqa: F401
        from aerial_gym.config.env_config.empty_env import EmptyEnvCfg
        from aerial_gym.registry.robot_registry import robot_registry
        from aerial_gym.utils import math as ref_math

        from . import hp1_oracle as O

        self.torch, self.O, self.ref_math = torch, O, ref_math
        self.N, self.episode_len_steps = int(num_envs), int(episode_len_steps)
        n = self.N

        class _E(EmptyEnvCfg):
            class env(EmptyEnvCfg.env):
                num_envs = n

        torch.manual_seed(seed)
        self.robot, self.cfg = robot_registry.make_robot("base_quadrotor", "lee_attitude_control", _E, "cpu")
        self.model = O.Hp1Model()  # mass / inertia / link transforms of quad.urdf (the reference takes them from Isaac Gym)
        rootst = torch.zeros(n, 13)
        rootst[:, 6] = 1.0
        B = 9  # quad.urdf: 9 links
        self.gtd = {
            "dt": 0.01, "gravity": torch.tensor([0.0, 0.0, -9.81]).expand(n, -1), "robot_state_tensor": rootst,
            "robot_position": rootst[:, 0:3], "robot_orientation": rootst[:, 3:7], "robot_linvel": rootst[:, 7:10],
            "robot_angvel": rootst[:, 10:13], "robot_force_tensor": torch.zeros(n, B, 3), "robot_torque_tensor": torch.zeros(n, B, 3),
            "env_bounds_min": -torch.ones(n, 3), "env_bounds_max": torch.ones(n, 3), "robot_mass": torch.full((n,), self.model.mass),
            "robot_inertia": torch.tensor(np.asarray(self.model.inertia), dtype=torch.float32).expand(n, -1, -1).clone(),
        }
        self.robot.init_tensors(self.gtd)
        self.mask = [int(x) for x in self.robot.application_mask.tolist()]
        self.compute_reward = _reference_compute_reward(root)
        self.sim_steps = torch.zeros(n, dtype=torch.int32)
        self.target = torch.zeros(n, 3)
        self.crashes = torch.zeros(n, dtype=torch.bool)
        self.truncations = torch.zeros(n, dtype=torch.bool)
        self.prev_actions = torch.zeros(n, 4)
        self.obs = torch.zeros(n, 13)
        self.rewards = torch.zeros(n)
        ec = _E.env
        self._bounds = tuple(torch.tensor(v, dtype=torch.float32) for v in (ec.lower_bound_min, ec.lower_bound_max, ec.upper_bound_min, ec.upper_bound_max))
        self.reset_idx(torch.arange(n))

    def reset_idx(self, env_ids):
        torch, g = self.torch, self.gtd
        n = self.N
        # IsaacGymEnv.reset_idx: env bounds (IGE_env_manager.py:513-519), full-N draws then gather, like the reference
        lo = (self._bounds[1] - self._bounds[0]) * torch.rand(n, 3) + self._bounds[0]
        hi = (self._bounds[3] - self._bounds[2]) * torch.rand(n, 3) + self._bounds[2]
        g["env_bounds_min"][env_ids] = lo[env_ids]
        g["env_bounds_max"][env_ids] = hi[env_ids]
        self.robot.reset_idx(env_ids)  # the reference's own reset (state, gains, motor model) + update_states for all envs
        self.sim_steps[env_ids] = 0

    def step(self, actions):
        torch, O, g = self.torch, self.O, self.gtd
        self.robot.step(actions)  # reference: update_states -> controller -> allocation -> motor model -> drag (+ disturbance)
        F, T = O.link_wrenches_to_body(self.model, g["robot_force_tensor"][:, self.mask], g["robot_torque_tensor"][:, self.mask],
                                       g["robot_force_tensor"][:, 0], g["robot_torque_tensor"][:, 0])
        g["robot_state_tensor"][:] = O.rigid_body_integrate(self.model, g["robot_state_tensor"], F, T)  # stand-in for gym.simulate
        self.sim_steps += 1
        self.crashes[:] = False
        pos_err_vehicle = self.ref_math.quat_apply_inverse(g["robot_vehicle_orientation"], self.target - g["robot_position"])
        rew, crashes = self.compute_reward(pos_err_vehicle, g["robot_linvel"], g["robot_orientation"], g["robot_body_angvel"], self.crashes, 1.0,
                                           actions, self.prev_actions, {})
        self.rewards[:], self.crashes[:] = rew, crashes
        self.truncations[:] = self.sim_steps > self.episode_len_steps
        ids = (self.crashes | self.truncations).nonzero(as_tuple=False).squeeze(-1)
        if ids.numel():
            self.reset_idx(ids)
        self.prev_actions = actions
        o = self.obs
        o[:, 0:3] = self.target - g["robot_position"]
        o[:, 3:7] = g["robot_orientation"]
        o[:, 7:10] = g["robot_body_linvel"]
        o[:, 10:13] = g["robot_body_angvel"]
        return o, self.rewards, self.crashes, self.truncations


def time_reference(n_envs, steps, warmup, seed=0):
    """(env-steps/s, s per step, torch threads used) of the loop above, best torch thread count of a few"""
    import time

    import torch

    task = ReferencePositionTask(n_envs, seed=seed)
    task.sim_steps[:] = (torch.arange(n_envs) % 500).to(torch.int32)
    g = torch.Generator().manual_seed(seed)
    acts = [torch.rand(n_envs, 4, generator=g) * 2 - 1 for _ in range(8)]
    for i in range(max(1, warmup)):
        task.step(acts[i % 8])
    max_t = torch.get_num_threads()
    best = (max_t, float("inf"))
    for nt in sorted({max_t, max(1, max_t // 2), max(1, max_t // 4), min(max_t, 8)}, reverse=True):
        torch.set_num_threads(nt)
        task.step(acts[0])
        t0 = time.perf_counter()
        for i in range(2):
            task.step(acts[i % 8])
        dt_ = time.perf_counter() - t0
        if dt_ < best[1]:
            best = (nt, dt_)
    torch.set_num_threads(best[0])
    t0 = time.perf_counter()
    for i in range(steps):
        task.step(acts[i % 8])
    dt = time.perf_counter() - t0
    used = torch.get_num_threads()
    torch.set_num_threads(max_t)
    return n_envs * steps / dt, dt / steps, used
