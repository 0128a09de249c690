"""Host side of HP1: owns the device tensors (PyTorch = allocator + streams only) and calls the
C ABI (include/aerial_gym_b200.h) through ctypes.  No arithmetic of the hot path happens here.

``MultirotorSpec`` is the flat, already-resolved description of one robot x controller x sim
configuration (what the reference spreads over robot_config / controller_config / sim_config /
Isaac Gym asset properties).  ``Hp1Engine`` binds a spec to N environments on one GPU.
"""
from __future__ import annotations

import ctypes as C
import functools
import math
from dataclasses import dataclass, field
from typing import Optional

import numpy as np
import torch

from . import _lib
from ._lib import AgxHp1Buffers, AgxHp1Config, AgxHp1ResetDraws

try:
    from ._hostcall import step_at as _step_at
except ImportError as exc:
    raise _lib.AgxError(f"the _hostcall extension is not built ({exc}): build it with `python -m aerial_gym_simulator_b200._build`") from None

PI = math.pi


@dataclass
class MultirotorSpec:
    """Field names deliberately match ``oracle.hp1_oracle.Hp1Model`` so tests can build the
    checker from the same numbers (``dataclasses.asdict``)."""

    num_motors: int = 4
    controller: int = _lib.CTRL_ATTITUDE
    dt: float = 0.01
    gravity: tuple = (0.0, 0.0, -9.81)
    mass: float = 0.25
    inertia: np.ndarray = field(default_factory=lambda: np.diag([8.45e-4, 8.45e-4, 1.69e-3]))
    com: np.ndarray = field(default_factory=lambda: np.zeros(3))
    allocation_matrix: np.ndarray = None
    motor_directions: np.ndarray = None
    thrust_to_torque_ratio: float = 0.01
    force_application_level: str = "motor_link"
    link_r: np.ndarray = None
    link_R: np.ndarray = None
    use_rps: bool = True
    integration_scheme: str = "rk4"
    use_discrete_approximation: bool = True
    min_thrust: float = 0.0
    max_thrust: float = 2.0
    max_thrust_rate: float = 100000.0
    tau_inc_range: tuple = (0.04, 0.04)
    tau_dec_range: tuple = (0.04, 0.04)
    k_thrust_range: tuple = (0.00000926312, 0.00001826312)
    max_yaw_rate: float = PI / 3.0
    K_pos_range: tuple = ((2.0, 2.0, 1.0), (3.0, 3.0, 2.0))
    K_vel_range: tuple = ((2.0, 2.0, 2.0), (3.0, 3.0, 3.0))
    K_rot_range: tuple = ((0.8, 0.8, 0.4), (1.2, 1.2, 0.6))
    K_angvel_range: tuple = ((0.1, 0.1, 0.1), (0.2, 0.2, 0.2))
    randomize_params: bool = False
    drag_lin1: tuple = (0.0, 0.0, 0.0)
    drag_lin2: tuple = (0.0, 0.0, 0.0)
    drag_ang1: tuple = (0.0, 0.0, 0.0)
    drag_ang2: tuple = (0.0, 0.0, 0.0)
    enable_disturbance: bool = False
    prob_apply_disturbance: float = 0.02
    max_disturbance: tuple = (0.75, 0.75, 0.75, 0.004, 0.004, 0.004)
    linear_damping: float = 0.01
    angular_damping: float = 0.01
    max_linear_velocity: float = 100.0
    max_angular_velocity: float = 100.0
    gyroscopic: bool = True
    min_init_state: tuple = (0.1, 0.15, 0.15, 0, 0, -PI / 6, 1.0, -0.2, -0.2, -0.2, -0.2, -0.2, -0.2)
    max_init_state: tuple = (0.2, 0.85, 0.85, 0, 0, PI / 6, 1.0, 0.2, 0.2, 0.2, 0.2, 0.2, 0.2)
    bounds_lower_range: tuple = ((-1.0, -1.0, -1.0), (-1.0, -1.0, -1.0))
    bounds_upper_range: tuple = ((1.0, 1.0, 1.0), (1.0, 1.0, 1.0))

    def __post_init__(self):
        M = self.num_motors
        if self.allocation_matrix is None:  # base_quad_config.py:166-173
            self.allocation_matrix = [
                [0.0, 0.0, 0.0, 0.0], [0.0, 0.0, 0.0, 0.0], [1.0, 1.0, 1.0, 1.0],
                [-0.13, -0.13, 0.13, 0.13], [-0.13, 0.13, 0.13, -0.13], [-0.01, 0.01, -0.01, 0.01],
            ]
        if self.motor_directions is None:
            self.motor_directions = [1, -1, 1, -1]
        if self.link_r is None:  # resources/robots/quad/quad.urdf joints base_link_to_motor_{0..3}
            self.link_r = [[0.13, -0.13, 0.0], [-0.13, -0.13, 0.0], [-0.13, 0.13, 0.0], [0.13, 0.13, 0.0]]
        if self.link_R is None:
            self.link_R = np.tile(np.eye(3), (M, 1, 1))
        self.allocation_matrix = np.asarray(self.allocation_matrix, dtype=np.float64)
        self.motor_directions = np.asarray(self.motor_directions, dtype=np.float64)
        self.link_r = np.asarray(self.link_r, dtype=np.float64)
        self.link_R = np.asarray(self.link_R, dtype=np.float64)
        self.inertia = np.asarray(self.inertia, dtype=np.float64)
        self.com = np.asarray(self.com, dtype=np.float64)
        if self.allocation_matrix.shape != (6, M):
            raise ValueError("Allocation matrix must have 6 rows and num_motors columns.")

    @property
    def num_actions(self) -> int:
        if self.controller == _lib.CTRL_NONE:
            return self.num_motors
        return 7 if self.controller == _lib.CTRL_FULLY_ACTUATED else 4

    def wrench_map(self) -> np.ndarray:
        """[6,M] motor thrust -> base-frame wrench about the COM (SURVEY Appendix B):
        motor_link: per-link local force [0,0,f], torque -cq*dir*[0,0,f] (control_allocation.py:103-114)
        carried through the fixed URDF transform of link i; otherwise the allocation matrix at body 0."""
        M = self.num_motors
        if self.force_application_level == "motor_link":
            W = np.zeros((6, M))
            for i in range(M):
                ez = self.link_R[i] @ np.array([0.0, 0.0, 1.0])
                W[0:3, i] = ez
                W[3:6, i] = np.cross(self.link_r[i] - self.com, ez) - self.thrust_to_torque_ratio * self.motor_directions[i] * ez
            return W
        W = self.allocation_matrix.copy()
        for i in range(M):
            W[3:6, i] += np.cross(-self.com, W[0:3, i])
        return W

    def alloc_pinv(self) -> np.ndarray:
        # torch.linalg.pinv of the fp32 matrix, as control_allocation.py:46-48 does
        A = torch.tensor(self.allocation_matrix, dtype=torch.float32)
        return torch.linalg.pinv(A).double().numpy()


@dataclass
class ArticulationSpec:
    """The joint layer of an articulated multirotor (DESIGN.md "Articulated robots"): the merged body table of its URDF
    (urdf.ArticulatedBodies), the drive gains per DOF, where each motor sits, and the ranges the joint state is reset to.
    The MultirotorSpec beside it keeps the zero-configuration mass and inertia, which is what the controller uses.
    drive_mode: per DOF (a scalar applies to all) "position" -- the implicit drive towards the setpoints -- or "effort" -- no drive
    (its stiffness and damping are set to 0 here; the URDF <dynamics damping> stays), the engine's dof_actuation_force instead,
    clamped to +-effort_limit where that is > 0.  effort_limit: [D] N m, default the URDF's <limit effort>.
    The units are per DOF: a prismatic DOF (bodies.joint_kinds) has q in m, k in N / m, d in N s / m, effort and effort_limit in N."""

    bodies: object                     # urdf.ArticulatedBodies
    stiffness: np.ndarray              # [D] k, N m / rad (N / m for a prismatic DOF)
    damping: np.ndarray                # [D] d, N m s / rad or N s / m (the URDF <dynamics damping> is added on top)
    motor_body: np.ndarray             # [M] body of each motor's application_mask link
    motor_R: np.ndarray                # [M,3,3] motor link frame in its body's frame
    motor_p: np.ndarray                # [M,3]
    motor_torque: np.ndarray           # [M] reaction torque per unit thrust about the motor z axis: -thrust_to_torque_ratio * dir
    init_dof_pos_range: tuple = None   # ([D], [D]) uniform reset range of q; default (0, 0)
    init_dof_vel_range: tuple = None   # ([D], [D]) of q-dot
    drive_mode: object = "position"    # [D] or scalar: "position" | "effort"
    effort_limit: np.ndarray = None    # [D] N m, |tau_e| bound of an effort DOF where > 0

    def __post_init__(self):
        b, D = self.bodies, self.bodies.num_dofs
        z = np.zeros(D)
        self.stiffness = np.broadcast_to(np.asarray(self.stiffness, np.float64), (D,)).copy()
        self.damping = np.broadcast_to(np.asarray(self.damping, np.float64), (D,)).copy()
        if (self.stiffness < 0).any() or (self.damping < 0).any():
            raise ValueError("joint stiffness and damping must be >= 0")
        mode = [self.drive_mode] * D if isinstance(self.drive_mode, str) else list(self.drive_mode)
        if len(mode) != D or any(m not in ("position", "effort") for m in mode):
            raise ValueError(f"drive_mode must be 'position' or 'effort', or a list of {D} of them (one per DOF); got {self.drive_mode!r}")
        self.drive_mode = mode
        self.effort_dof = np.array([m == "effort" for m in mode], bool)
        self.effort_limit = np.broadcast_to(np.asarray(b.effort_limit[1:] if self.effort_limit is None else self.effort_limit, np.float64),
                                            (D,)).copy()
        if not (self.effort_limit >= 0).all():
            raise ValueError("effort_limit must be >= 0")
        self.stiffness[self.effort_dof] = 0.0  # an effort DOF has no implicit drive
        self.damping[self.effort_dof] = 0.0
        rng = lambda r: (z.copy(), z.copy()) if r is None else tuple(np.broadcast_to(np.asarray(v, np.float64), (D,)).copy() for v in r)
        self.init_dof_pos_range, self.init_dof_vel_range = rng(self.init_dof_pos_range), rng(self.init_dof_vel_range)
        self.motor_body = np.asarray(self.motor_body, np.int64)
        self.motor_R, self.motor_p = np.asarray(self.motor_R, np.float64), np.asarray(self.motor_p, np.float64)
        self.motor_torque = np.asarray(self.motor_torque, np.float64)
        # a movable subtree without inertia about its axis (a slider's: without mass) and without a drive would make the joint's pivot
        # D_i zero
        d_tot = self.damping + b.urdf_damping[1:]
        R0, P0 = [np.eye(3)], [np.zeros(3)]
        for i in range(1, b.num_bodies):
            l = b.parent[i]
            R0.append(R0[l] @ b.joint_R[i])
            P0.append(P0[l] + R0[l] @ b.joint_p[i])
        for i in range(1, b.num_bodies):
            if self.stiffness[i - 1] > 0 or d_tot[i - 1] > 0:
                continue
            a = R0[i] @ b.axis[i]
            slide = b.joint_kinds[i] == "prismatic"
            J = 0.0
            for k in range(i, b.num_bodies):
                anc = k
                while anc > i:
                    anc = b.parent[anc]
                if anc != i:
                    continue
                if slide:  # S = (0, a): S^T I S is the subtree's mass
                    J += float(b.mass[k])
                    continue
                r = P0[k] + R0[k] @ b.com[k] - P0[i]
                Ic = R0[k] @ b.inertia[k] @ R0[k].T + b.mass[k] * (float(r @ r) * np.eye(3) - np.outer(r, r))
                J += float(a @ Ic @ a)
            if not J > 1e-12:
                why = "it is in effort mode and has no URDF <dynamics damping>" if self.effort_dof[i - 1] else \
                    "stiffness = damping = 0"
                what = "no mass to slide" if slide else "no inertia about the axis"
                raise ValueError(f"joint '{b.joint_names[i]}': its subtree has {what} and the joint has no drive "
                                 f"({why}), so its acceleration is undefined")

    @property
    def num_dofs(self) -> int:
        return self.bodies.num_dofs

    def prismatic_mask(self) -> int:
        """the joint kinds for agx_hp1_articulated_step_prismatic: bit i set = body i's joint is prismatic (0: no prismatic joint)"""
        return sum(1 << i for i, k in enumerate(self.bodies.joint_kinds) if k == "prismatic")

    def effort_struct(self) -> "_lib.AgxJointEffort":
        """the AgxJointEffort of the effort DOFs (its `effort` pointer left NULL)"""
        e = _lib.AgxJointEffort()
        for j in range(self.num_dofs):
            e.effort_dof[j + 1] = int(self.effort_dof[j])
            e.effort_limit[j + 1] = float(self.effort_limit[j])
        return e

    def to_struct(self) -> "_lib.AgxArticulation":
        b, a = self.bodies, _lib.AgxArticulation()
        a.num_bodies, a.num_dofs = b.num_bodies, b.num_dofs
        for i in range(b.num_bodies):
            a.parent[i] = int(b.parent[i])
            _set(a.joint_R[i], b.joint_R[i]); _set(a.joint_p[i], b.joint_p[i]); _set(a.axis[i], b.axis[i])
            a.mass[i] = float(b.mass[i])
            _set(a.com[i], b.com[i]); _set(a.inertia[i], b.inertia[i])
            a.lower[i], a.upper[i], a.limited[i] = float(b.lower[i]), float(b.upper[i]), int(bool(b.limited[i]))
            if i > 0:
                a.stiffness[i] = float(self.stiffness[i - 1])
                a.damping[i] = float(self.damping[i - 1] + b.urdf_damping[i])
        for k in range(len(self.motor_body)):
            a.motor_body[k] = int(self.motor_body[k])
            _set(a.motor_R[k], self.motor_R[k]); _set(a.motor_p[k], self.motor_p[k])
            a.motor_torque[k] = float(self.motor_torque[k])
        return a


def _set(arr, vals):
    vals = np.asarray(vals, dtype=np.float64).reshape(-1)
    for i, v in enumerate(vals):
        arr[i] = float(v)


def build_config(spec: MultirotorSpec, num_envs: int, *, physics_steps=1, episode_len_steps=500, seed=0,
                 env_id_offset=0, device_rng_reset=True, strict_stale_obs=True, crash_distance=8.0) -> AgxHp1Config:
    c = AgxHp1Config()
    M = spec.num_motors
    c.num_envs, c.num_motors, c.controller, c.num_actions = num_envs, M, spec.controller, spec.num_actions
    c.physics_steps, c.episode_len_steps, c.env_id_offset = physics_steps, episode_len_steps, env_id_offset
    c.seed = seed & 0xFFFFFFFFFFFFFFFF
    flags = 0
    flags |= _lib.F_USE_RPS if spec.use_rps else 0
    flags |= _lib.F_MOTOR_RK4 if spec.integration_scheme != "euler" else 0
    flags |= _lib.F_DISCRETE_MIX if spec.use_discrete_approximation else 0
    flags |= _lib.F_GYROSCOPIC if spec.gyroscopic else 0
    flags |= _lib.F_RANDOMIZE_GAINS if spec.randomize_params else 0
    flags |= _lib.F_DEVICE_RNG_RESET if device_rng_reset else 0
    flags |= _lib.F_STRICT_STALE_OBS if strict_stale_obs else 0
    c.flags = flags
    c.dt, c.mass = spec.dt, spec.mass
    _set(c.gravity, spec.gravity)
    _set(c.inertia, spec.inertia)
    _set(c.inertia_inv, np.linalg.inv(spec.inertia))
    _set(c.alloc_pinv, spec.alloc_pinv())  # [M,6] row-major
    W = np.zeros((6, _lib.AGX_MAX_MOTORS))
    W[:, :M] = spec.wrench_map()
    _set(c.wrench_map, W)
    _set(c.com, spec.com)
    c.min_thrust, c.max_thrust, c.max_thrust_rate = spec.min_thrust, spec.max_thrust, spec.max_thrust_rate
    c.max_yaw_rate = spec.max_yaw_rate
    _set(c.drag_lin1, spec.drag_lin1); _set(c.drag_lin2, spec.drag_lin2)
    _set(c.drag_ang1, spec.drag_ang1); _set(c.drag_ang2, spec.drag_ang2)
    c.linear_damping, c.angular_damping = spec.linear_damping, spec.angular_damping
    c.max_linear_velocity, c.max_angular_velocity = spec.max_linear_velocity, spec.max_angular_velocity
    # construction-time gains: mid-point of min/max in fp32 (base_lee_controller.py:59-62)
    mid = lambda r: ((np.float32(r[1]) + np.float32(r[0])) / np.float32(2.0)).astype(np.float64)
    f32a = lambda x: np.asarray(x, dtype=np.float32)
    _set(c.K_pos, mid((f32a(spec.K_pos_range[0]), f32a(spec.K_pos_range[1]))))
    _set(c.K_vel, mid((f32a(spec.K_vel_range[0]), f32a(spec.K_vel_range[1]))))
    _set(c.K_rot, mid((f32a(spec.K_rot_range[0]), f32a(spec.K_rot_range[1]))))
    _set(c.K_angvel, mid((f32a(spec.K_angvel_range[0]), f32a(spec.K_angvel_range[1]))))
    c.tau_inc, c.tau_dec, c.k_thrust = spec.tau_inc_range[0], spec.tau_dec_range[0], spec.k_thrust_range[0]
    c.crash_distance = crash_distance
    c.dist_prob = float(spec.prob_apply_disturbance)
    _set(c.dist_max, spec.max_disturbance)
    c.dist_seed = (int(seed) ^ 0xD157_0000_D157) & 0xFFFFFFFFFFFFFFFF  # the stream EnvManager._draw_disturbance uses for agx_disturbance_draw
    _set(c.min_init_state, spec.min_init_state); _set(c.max_init_state, spec.max_init_state)
    _set(c.bounds_lo_min, spec.bounds_lower_range[0]); _set(c.bounds_lo_max, spec.bounds_lower_range[1])
    _set(c.bounds_hi_min, spec.bounds_upper_range[0]); _set(c.bounds_hi_max, spec.bounds_upper_range[1])
    _set(c.tau_inc_range, spec.tau_inc_range); _set(c.tau_dec_range, spec.tau_dec_range)
    _set(c.k_thrust_range, spec.k_thrust_range)
    _set(c.K_pos_min, spec.K_pos_range[0]); _set(c.K_pos_max, spec.K_pos_range[1])
    _set(c.K_vel_min, spec.K_vel_range[0]); _set(c.K_vel_max, spec.K_vel_range[1])
    _set(c.K_rot_min, spec.K_rot_range[0]); _set(c.K_rot_max, spec.K_rot_range[1])
    _set(c.K_angvel_min, spec.K_angvel_range[0]); _set(c.K_angvel_max, spec.K_angvel_range[1])
    return c


_raw_stream = getattr(torch._C, "_cuda_getCurrentRawStream", None)


class Hp1Engine:
    """N environments of one MultirotorSpec on one CUDA device.

    per_env_params: "auto" allocates a per-env array only for parameters whose reset range is
    non-degenerate (they must be streamed); "all" allocates every array (needed to inject
    arbitrary values, e.g. in parity tests)."""

    DERIVED = ("euler", "vehicle_orientation", "vehicle_linvel", "body_linvel", "body_angvel")

    def __init__(self, spec: MultirotorSpec, num_envs: int, device="cuda:0", *, physics_steps=1,
                 episode_len_steps=500, seed=0, env_id_offset=0, device_rng_reset=True, strict_stale_obs=True,
                 materialize_derived=True, per_env_params="auto", debug_wrench=False, host_io=False, articulation=None,
                 imu_body=None, joint_force=False):
        """host_io: obs / reward / terminations / truncations live in pinned, device-mapped HOST
        memory (agx_host_alloc) and the fused task step stores them there directly over PCIe;
        `actions` may then be a pinned host tensor (e.g. `self.host_actions`) that the kernel
        reads in place.  The caller synchronises the stream before reading the results.
        articulation: an ArticulationSpec -- the robot has joints; physics_step runs agx_hp1_articulated_step and the engine owns
        dof_state [N,D,2] and the drive targets dof_position_setpoint / dof_velocity_setpoint [N,D] (zero until the caller writes
        them), and body_state [N,B,13], every body's pose and velocity, which update_body_state() refreshes.  There is no fused task
        step for such a robot.
        imu_body: with an articulation, the body an IMU rides on -- physics_step then runs agx_hp1_articulated_step_imu, which also
        writes imu_input [N,9] = (force f_b, torque n_b, angular velocity w_b) of that body in its own frame, of the last
        sub-step's start (the IMU's force input; the state update is the same arithmetic).
        An articulation with a DOF in effort mode (ArticulationSpec.drive_mode): the engine also owns dof_actuation_force [N,D],
        the commanded joint torques, zero until the caller writes them and never written by the engine; physics_step then runs
        agx_hp1_articulated_step_effort, which reads it in place once per launch (the columns of position DOFs are ignored).
        joint_force: with an articulation, the engine also owns joint_wrench [N,B,6] and dof_force [N,D], zero until the first step;
        physics_step then runs agx_hp1_articulated_step_joint_force (with the IMU input and the effort DOFs above, if any), which
        writes them from the last sub-step: row i >= 1 of joint_wrench is the force and the torque (about the joint origin) body i's
        parent exerts on it through joint i, both in body i's frame, row 0 is zero; dof_force is each joint's torque along its axis.
        An articulation with a prismatic joint runs agx_hp1_articulated_step_prismatic (with the IMU input, the effort DOFs and the
        joint forces above, as configured) and agx_hp1_articulated_body_state_prismatic instead; its prismatic DOFs hold metres in
        dof_state and the setpoints, N in dof_actuation_force and dof_force (the force along the slide)."""
        self.lib = _lib.load()
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise _lib.AgxError("Hp1Engine needs a CUDA device: there is no CPU path")
        self._init_articulation(articulation, num_envs, debug_wrench, host_io)
        self.spec, self.N, self.M = spec, int(num_envs), spec.num_motors
        self.cfg = build_config(spec, self.N, physics_steps=physics_steps, episode_len_steps=episode_len_steps,
                                seed=seed, env_id_offset=env_id_offset, device_rng_reset=device_rng_reset,
                                strict_stale_obs=strict_stale_obs)
        N, M, dev = self.N, self.M, self.device
        self._init_body_state()
        self._init_imu(imu_body)
        self._init_effort()
        self._init_joint_force(joint_force)
        z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device=dev)
        self.root_state = z(N, 13)
        self.root_state[:, 6] = 1.0
        self.motor_thrust = z(N, M)
        self.sim_steps = z(N, dt=torch.int32)
        self.target_position = z(N, 3)
        self.host_io, self._host_allocs = bool(host_io), []
        if self.host_io:
            self.obs = self._host_tensor((N, 13), torch.float32)
            self.reward = self._host_tensor((N,), torch.float32)
            self.terminations = self._host_tensor((N,), torch.bool)
            self.truncations = self._host_tensor((N,), torch.bool)
            self.host_actions = self._host_tensor((N, spec.num_actions), torch.float32)
        else:
            self.obs = z(N, 13)
            self.reward = z(N)
            self.terminations = z(N, dt=torch.bool)
            self.truncations = z(N, dt=torch.bool)
        self.reset_mask = z(N, dt=torch.bool)
        self.any_reset = z(32, dt=torch.int32)
        self.tile_sync = z(2 * ((N + 31) // 32), dt=torch.int32)  # per-tile claim / done counters (chained steps)
        self.publish_ctr = z(16, dt=torch.int64)  # [0..3] published-tile counters (a 128-byte line of their own), used while a gather is attached
        self.episode_count = z(N, dt=torch.int32)
        self.bounds_min = torch.tensor(spec.bounds_lower_range[0], dtype=torch.float32, device=dev).expand(N, -1).clone()
        self.bounds_max = torch.tensor(spec.bounds_upper_range[0], dtype=torch.float32, device=dev).expand(N, -1).clone()
        allp = per_env_params == "all"
        nd = lambda r: allp or (np.asarray(r[0]) != np.asarray(r[1])).any()
        full = lambda v, *s: torch.full(s, float(v), dtype=torch.float32, device=dev)
        self.tau_inc = full(spec.tau_inc_range[0], N, M) if nd(spec.tau_inc_range) else None
        self.tau_dec = full(spec.tau_dec_range[0], N, M) if nd(spec.tau_dec_range) else None
        self.k_thrust = full(spec.k_thrust_range[0], N, M) if (spec.use_rps and nd(spec.k_thrust_range)) else None
        gains = allp or spec.randomize_params
        gk = lambda a: torch.tensor([a[i] for i in range(3)], dtype=torch.float32, device=dev).expand(N, -1).clone()
        self.K_pos = gk(self.cfg.K_pos) if gains else None
        self.K_vel = gk(self.cfg.K_vel) if gains else None
        self.K_rot = gk(self.cfg.K_rot) if gains else None
        self.K_angvel = gk(self.cfg.K_angvel) if gains else None
        self.euler = z(N, 3) if materialize_derived else None
        self.vehicle_orientation = z(N, 4) if materialize_derived else None
        self.vehicle_linvel = z(N, 3) if materialize_derived else None
        self.body_linvel = z(N, 3) if materialize_derived else None
        self.body_angvel = z(N, 3) if materialize_derived else None
        self.body_wrench = z(N, 6) if debug_wrench else None
        # scratch for the light obs patch (only useful when derived states are not materialised)
        self.fresh_vel = z(6, N) if (strict_stale_obs and not materialize_derived) else None
        self._actions_ok = {}
        self._gather, self.gathered_obs, self._own_obs = None, None, self.obs
        self._buf = AgxHp1Buffers()
        self._sync_buffers()
        self._cfg_ref, self._buf_ref = C.byref(self.cfg), C.byref(self._buf)
        # number of single-launch (chained) task steps since tile_sync / any_reset were zeroed = the step index the kernel's
        # per-tile claim counters hand out; the gather's push waits on that step's arrival counter
        self._chain_T = 0
        self._chain_counts = bool(self.lib.agx_hp1_task_step_is_chained(self._cfg_ref, self._buf_ref))
        self._dev_index = self.device.index if self.device.index is not None else torch.cuda.current_device()
        # agx_hp1_position_task_step_at(cfg, buf, stream, step_index), the structs passed by address, through the _hostcall extension:
        # the call is made every step, and a ctypes call costs ~10x as much host time
        self._task_step_at = functools.partial(_step_at, C.cast(self.lib.agx_hp1_position_task_step_at, C.c_void_p).value)
        self._cfg_addr, self._buf_addr = C.addressof(self.cfg), C.addressof(self._buf)
        self._task_step_gathered = self.lib.agx_hp1_position_task_step_gathered
        self._plain = self.art is None  # no gather attached, no disturbance buffer or counter set: position_task_step's fast path

    # ---- plumbing ---------------------------------------------------------------------------
    def _art_step_args(self):
        """(name, arguments but the stream) of the articulated step entry physics_step runs for this robot, from the engine's state
        at the call: with joint_force, the joint-force step (with the IMU input and the effort DOFs, if any); else with an effort
        table, the effort step (with the IMU input, if any); else with imu_body, the IMU step; else the plain step.  A robot with a
        prismatic joint takes the prismatic step, with whichever of these it has"""
        head = (self._cfg_ref, self._buf_ref, self._art_ref)
        imu = (self.imu_body, self.imu_input.data_ptr()) if self.imu_input is not None else (0, None)
        if self._prismatic:  # a robot with a prismatic joint: one entry for every combination of the above
            effort = self._effort_ref if self._effort is not None else None
            out = (self.joint_wrench.data_ptr(), self.dof_force.data_ptr()) if self.joint_wrench is not None else (None, None)
            return "agx_hp1_articulated_step_prismatic", head + (self._prismatic, effort) + imu + out
        if self.joint_wrench is not None:
            effort = self._effort_ref if self._effort is not None else None
            out = (self.joint_wrench.data_ptr(), self.dof_force.data_ptr())
            return "agx_hp1_articulated_step_joint_force", head + (effort,) + imu + out
        if self._effort is not None:
            return "agx_hp1_articulated_step_effort", head + (self._effort_ref,) + imu
        if self.imu_input is not None:
            return "agx_hp1_articulated_step_imu", head + imu
        return "agx_hp1_articulated_step", head

    def _init_articulation(self, articulation, num_envs, debug_wrench, host_io):
        self.articulation, self.art, self._prismatic = articulation, None, 0
        self.dof_state = self.dof_position_setpoint = self.dof_velocity_setpoint = None
        if articulation is None:
            return
        self._prismatic = articulation.prismatic_mask()
        if debug_wrench:
            raise ValueError("an articulated robot has no single body wrench to report (debug_wrench)")
        if host_io:
            raise NotImplementedError("host_io is a feature of the fused task step, which articulated robots do not have")
        N, D, dev = int(num_envs), articulation.num_dofs, self.device
        self.dof_state = torch.zeros(N, D, 2, dtype=torch.float32, device=dev)
        self.dof_position_setpoint = torch.zeros(N, D, dtype=torch.float32, device=dev)
        self.dof_velocity_setpoint = torch.zeros(N, D, dtype=torch.float32, device=dev)
        self.art = articulation.to_struct()
        self.art.dof_state = self.dof_state.data_ptr()
        self.art.dof_position_setpoint = self.dof_position_setpoint.data_ptr()
        self.art.dof_velocity_setpoint = self.dof_velocity_setpoint.data_ptr()
        self._art_ref = C.byref(self.art)

    def _init_body_state(self):
        """body_state [N,B,13] of an articulated robot (None otherwise), zero until update_body_state()"""
        self.body_state = None
        if self.articulation is not None:
            B = self.articulation.bodies.num_bodies
            self.body_state = torch.zeros(self.N, B, 13, dtype=torch.float32, device=self.device)

    def _init_imu(self, imu_body):
        """imu_input [N,9] of an articulated robot with an IMU on body imu_body (None otherwise), zero until the first step"""
        self.imu_body, self.imu_input = None, None
        if imu_body is None:
            return
        if self.articulation is None:
            raise ValueError("imu_body belongs to an articulated robot (Hp1Engine(articulation=...)): a rigid robot's IMU reads "
                             "body_wrench (debug_wrench=True)")
        self.imu_body = int(imu_body)
        self.imu_input = torch.zeros(self.N, 9, dtype=torch.float32, device=self.device)

    def _init_effort(self):
        """dof_actuation_force [N,D] and the AgxJointEffort of an articulated robot with an effort DOF (None otherwise)"""
        self.dof_actuation_force, self._effort = None, None
        if self.articulation is None or not self.articulation.effort_dof.any():
            return
        self.dof_actuation_force = torch.zeros(self.N, self.articulation.num_dofs, dtype=torch.float32, device=self.device)
        self._effort = self.articulation.effort_struct()
        self._effort.effort = self.dof_actuation_force.data_ptr()
        self._effort_ref = C.byref(self._effort)

    def _init_joint_force(self, joint_force):
        """joint_wrench [N,B,6] and dof_force [N,D] of an articulated robot with joint_force (None otherwise), zero until the first step"""
        self.joint_wrench, self.dof_force = None, None
        if not joint_force:
            return
        if self.articulation is None:
            raise ValueError("joint_force belongs to an articulated robot (Hp1Engine(articulation=...)): a rigid robot has no joints to "
                             "sense")
        B, D = self.articulation.bodies.num_bodies, self.articulation.num_dofs
        self.joint_wrench = torch.zeros(self.N, B, 6, dtype=torch.float32, device=self.device)
        self.dof_force = torch.zeros(self.N, D, dtype=torch.float32, device=self.device)

    def _host_tensor(self, shape, dtype):
        nbytes = max(1, int(np.prod(shape))) * torch.empty((), dtype=dtype).element_size()
        p = C.c_void_p()
        _lib.check(self.lib.agx_host_alloc(nbytes, C.byref(p)), "agx_host_alloc")
        raw = (C.c_uint8 * nbytes).from_address(p.value)
        C.memset(p, 0, nbytes)
        self._host_allocs.append((p, raw))
        n = int(np.prod(shape))
        if n == 0:
            return torch.empty(shape, dtype=dtype)
        return torch.frombuffer(raw, dtype=dtype, count=n).view(shape)

    def close(self):
        """Free the mapped host buffers (host_io).  The tensors handed out must not be used afterwards."""
        torch.cuda.synchronize(self.device)
        for p, _ in self._host_allocs:
            self.lib.agx_host_free(p)
        self._host_allocs = []

    def _ptr(self, t: Optional[torch.Tensor]):
        return None if t is None else t.data_ptr()

    def _sync_buffers(self):
        b = self._buf
        for name in _lib._HP1_BUF_FIELDS:
            if name in ("actions", "disturbance", "dist_counter", "dist_offset_", "publish_ctr"):
                continue
            setattr(b, name, self._ptr(getattr(self, name, None)))

    def attach_obs_gather(self, gather):
        """Run the multi-GPU observation all-gather BESIDE the task steps (distributed.PipelinedObsGather, SURVEY 8e).

        The step kernel itself never touches NVLink.  While a gather is attached, `position_task_step` writes this rank's
        observation straight into its slot of the next buffer of the gather's ring (`self.obs` is a view of that slot) and
        enqueues the push kernel (NVLink peer stores + per-peer flags) on the ring slot's side stream; on the chained single-launch
        path the push waits for the step's completion counter in device memory, so nothing is recorded between the chained
        launches and the push of step t overlaps the compute of the following steps (a step only waits -- by a stream event, on
        the host's initiative -- when the push that last read its ring slot is still running).
        `self.gathered_obs` is the [world*N, 13] buffer of the last step: complete after `gather.wait()` (a tiny kernel on the
        current stream that retires when every rank's rows have landed).  Several engines may share one gather object."""
        if gather is not None and gather.bytes != self.N * 13 * 4:
            raise ValueError("gather object was built for a different shard size")
        if gather is not None and self.host_io:
            raise ValueError("host_io and an attached observation gather are mutually exclusive (obs lives in the gather ring)")
        if self._gather is not None and gather is None:
            self._gather.fence()
            self.obs, self._buf.obs = self._own_obs, self._own_obs.data_ptr()
            self._buf.publish_ctr = None
        self._gather, self.gathered_obs = gather, None
        self._plain = False  # the next position_task_step takes the full path, which sets it again
        if gather is not None:
            # four u64 published-tile counters on a line of their own, switched on only while a gather is attached; they must agree with
            # the step index, so attaching is a quiet point: drain, zero them and restart the chain's step numbering
            self._rebase_chain()
            self._buf.publish_ctr = self.publish_ctr.data_ptr()
            self._ready_base = self.publish_ctr.data_ptr()
            self._n_tiles = (self.N + 31) // 32

    def _arm_gather(self, chained):
        """before the launch: this step's observation goes into the ring slot of the next epoch"""
        g = self._gather
        epoch, slot = g.next_epoch()
        self.obs = g.own_slot[slot]
        self._buf.obs = g.own_slot_ptr[slot]
        return epoch, slot

    def _push_gather(self, chained, epoch, slot):
        """after the launch: the push of this step's rows"""
        g = self._gather
        if chained:
            T = self._chain_T
            g.push(self._buf.obs, epoch, slot, ready_ctr=self._ready_base + 8 * (T & 3), ready_target=(T // 4 + 1) * self._n_tiles)
        else:
            g.push(self._buf.obs, epoch, slot, stream=self._stream())  # two-launch path: plain stream order
        self.gathered_obs = g.outs[slot]

    CHAIN_REBASE_STEPS = 1 << 30  # the kernel's step index, flags and per-tile counters are 32-bit: rebased long before they wrap (~3 h at 10 us / step)

    def _rebase_chain(self):
        """zero the chained step's counters at a quiet point (stream drained, pushes finished) and restart the step index at 0"""
        if self._gather is not None:
            self._gather.fence()
        torch.cuda.current_stream(self.device).synchronize()
        err = int(self.any_reset[2].item())
        self.tile_sync.zero_()
        self.any_reset[4:].zero_()
        self.publish_ctr.zero_()
        self.any_reset[2] = err
        self._chain_T = 0

    def check(self):
        """Synchronise the current stream and raise if a bounded in-kernel wait of the chained step expired (AGX_E_TIMEOUT)."""
        _lib.check(self.lib.agx_hp1_check(self._buf_ref, self._stream()), "agx_hp1_check")

    def _stream(self):
        # raw stream handle of torch's current stream (the fast private getter when available: the
        # step is ~12 us of GPU time, every microsecond of host time per call counts)
        if _raw_stream is not None:
            return _raw_stream(self._dev_index)
        return torch.cuda.current_stream(self.device).cuda_stream

    def _check_actions(self, actions):
        key = id(actions)
        hit = self._actions_ok.get(key)
        if hit is not None and hit[0] is actions:
            self._buf.actions = hit[1]
            return
        if actions.shape != (self.N, self.cfg.num_actions):
            raise ValueError("Action tensor does not have the correct number of environments")
        on_host_ok = self.host_io and actions.device.type == "cpu" and (
            actions.data_ptr() == self.host_actions.data_ptr() or actions.is_pinned())
        if actions.dtype != torch.float32 or not actions.is_contiguous() or not (actions.device == self.device or on_host_ok):
            raise ValueError("actions must be a contiguous float32 tensor on the engine's device"
                             + (" or in pinned host memory" if self.host_io else ""))
        if len(self._actions_ok) >= 32:
            self._actions_ok.clear()
        # validated tensors are remembered (with a reference, so the id cannot be recycled): shape,
        # dtype, device and storage of a live tensor object do not change under in-place writes
        self._actions_ok[key] = (actions, actions.data_ptr())
        self._buf.actions = actions.data_ptr()

    # ---- C ABI calls ------------------------------------------------------------------------
    def physics_step(self, actions, disturbance=None, physics_steps=None, dist_counter=None, dist_offset=0):
        """dist_counter: device uint32 tensor -- draw the disturbance inside the kernel (sub-step s uses draw counter
        *dist_counter + dist_offset + s; AgxHp1Buffers.dist_counter), instead of reading `disturbance` [N,6]"""
        self._check_actions(actions)
        self._plain = False
        self._buf.disturbance = self._ptr(disturbance)
        self._buf.dist_counter = None if (dist_counter is None or disturbance is not None) else dist_counter.data_ptr()
        self._buf.dist_offset = dist_offset
        if physics_steps is not None:
            self.cfg.physics_steps = int(physics_steps)
        if self.art is not None:
            name, args = self._art_step_args()
            _lib.check(getattr(self.lib, name)(*args, self._stream()), name)
            return
        _lib.check(self.lib.agx_hp1_physics_step(self._cfg_ref, self._buf_ref, self._stream()), "agx_hp1_physics_step")

    def update_body_state(self):
        """body_state [N,B,13] of an articulated robot from root_state and dof_state (agx_hp1_articulated_body_state): per body the
        world position of its frame origin, the xyzw quaternion body -> world, the world linear velocity of the origin and the world
        angular velocity; row 0 is root_state's.  One launch, no RNG, capturable."""
        if self.art is None:
            raise ValueError("body_state belongs to an articulated robot (Hp1Engine(articulation=...))")
        if self._prismatic:
            _lib.check(self.lib.agx_hp1_articulated_body_state_prismatic(
                self._art_ref, self._prismatic, self.N, self.root_state.data_ptr(), self.root_state.stride(0), self.body_state.data_ptr(),
                self._stream()), "agx_hp1_articulated_body_state_prismatic")
            return
        _lib.check(self.lib.agx_hp1_articulated_body_state(self._art_ref, self.N, self.root_state.data_ptr(), self.root_state.stride(0),
                                                           self.body_state.data_ptr(), self._stream()), "agx_hp1_articulated_body_state")

    def position_task_step(self, actions, disturbance=None, physics_steps=None, mid_event=None):
        """mid_event: optional torch.cuda.Event(enable_timing=True), already recorded once (so its
        handle exists); the library records it between the main kernel and the refresh pass."""
        if self._plain and disturbance is None and physics_steps is None and mid_event is None:
            # the common call -- an actions tensor validated before, nothing else -- in a straight line: the device takes ~10 us per
            # step, and a host that takes as long to enqueue it sets the pace.  The library reads the live cfg and buffers.
            hit = self._actions_ok.get(id(actions))
            T = self._chain_T
            if hit is not None and hit[0] is actions and T < self.CHAIN_REBASE_STEPS:
                self._buf.actions = hit[1]
                rc = self._task_step_at(self._cfg_addr, self._buf_addr, self._stream(), T)
                if rc:
                    _lib.check(rc, "agx_hp1_position_task_step_at")
                if self._chain_counts:
                    self._chain_T = T + 1
                return
        if self.art is not None:
            raise ValueError("an articulated robot has no fused task step: step it with physics_step (PositionSetpointTask does)")
        self._check_actions(actions)
        self._buf.disturbance = None if disturbance is None else disturbance.data_ptr()
        self._buf.dist_counter = None
        self._plain = disturbance is None and self._gather is None
        if physics_steps is not None:
            self.cfg.physics_steps = int(physics_steps)
        chained = self._chain_counts and mid_event is None  # which path the library takes for this launch
        if chained and self._chain_T >= self.CHAIN_REBASE_STEPS:
            self._rebase_chain()
        g = self._gather
        if g is not None and chained:
            # gate (ring slot free?) + step + push of its rows: one C call, three launches
            g.epoch += 1
            e, B = g.epoch, g.num_buffers
            slot = e % B
            own = g.own_slot_ptr[slot]
            self.obs, self._buf.obs = g.own_slot[slot], own
            a, ref = g._pushes[slot]
            T = self._chain_T
            a.local, a.epoch, a.ready_ctr, a.ready_target = own, e, self._ready_base + 8 * (T & 3), (T // 4 + 1) * self._n_tiles
            rc = self._task_step_gathered(self._cfg_ref, self._buf_ref, self._stream(), g._read_done_ptr[slot] if e > B else None, e - B,
                                          g._err_ptr, ref, g._raw[slot])
            if rc:
                _lib.check(rc, "agx_hp1_position_task_step_gathered")
            g._pending[slot] = True
            self.gathered_obs = g.outs[slot]
            self._chain_T = T + 1
            return
        armed = self._arm_gather(chained) if g is not None else None
        if mid_event is None:
            rc = self._task_step_at(self._cfg_addr, self._buf_addr, self._stream(), self._chain_T)
        else:
            rc = self.lib.agx_hp1_position_task_step_profiled(self._cfg_ref, self._buf_ref, self._stream(),
                                                              C.c_void_p(mid_event.cuda_event))
        if rc:
            _lib.check(rc, "agx_hp1_position_task_step")
        if armed is not None:
            self._push_gather(chained, *armed)
        if chained:
            self._chain_T += 1

    def reset(self, mask: torch.Tensor, draws: Optional[dict] = None):
        """mask: bool [N].  draws: dict of uniform [0,1) tensors keyed like AgxHp1ResetDraws, or None
        for the device RNG."""
        if mask.dtype != torch.bool or mask.shape != (self.N,):
            raise ValueError("mask must be bool [N]")
        d = None
        if draws is not None:
            d = AgxHp1ResetDraws()
            for k in _lib._HP1_DRAW_FIELDS:
                t = draws.get(k)
                if t is not None and (t.dtype != torch.float32 or not t.is_contiguous()):
                    raise ValueError(f"draw {k} must be contiguous float32")
                setattr(d, k, self._ptr(t))
        _lib.check(self.lib.agx_hp1_reset(C.byref(self.cfg), C.byref(self._buf), C.c_void_p(mask.data_ptr()),
                                          C.byref(d) if d is not None else None, self._stream()), "agx_hp1_reset")

    def refresh(self, only_if_flag=False):
        _lib.check(self.lib.agx_hp1_refresh(C.byref(self.cfg), C.byref(self._buf), int(only_if_flag), self._stream()),
                   "agx_hp1_refresh")
