"""HP1 oracle -- CPU restatement of the reference's dynamics/controller hot path.

TEST INFRASTRUCTURE ONLY.  Nothing under ``aerial_gym_simulator_b200/`` imports
this module; only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s
``cpu_baseline`` / ``--impl reference`` legs do, and only as the checker or the
reported CPU baseline -- never as the product path.

What it restates (reference = $AERIAL_GYM_REFERENCE/aerial_gym, commit f0d0f05):

* quaternion helpers                      utils/math.py:58-65, 123-180, 242-293, 313-347
* BaseMultirotor.update_states            robots/base_multirotor.py:287-294
* Lee controllers                         control/controllers/*.py, base_lee_controller.py:120-215
* ControlAllocator                        control/control_allocation.py:52-114
* MotorModel                              control/motor_model.py:88-251
* drag / disturbance                      robots/base_multirotor.py:213-285
* reset sampling                          robots/base_multirotor.py:177-205,
                                          control/motor_model.py:140-154,
                                          env_manager/IGE_env_manager.py:513-519,
                                          control/controllers/base_lee_controller.py:101-118
* position-task reward / obs              task/position_setpoint_task/position_setpoint_task.py:152-282
* env step bookkeeping                    env_manager/env_manager.py:342-432

PARITY PINNING.  Everything above is pinned against the reference's own torch
code imported in the build container (``tests/golden/make_golden.py`` writes the
fixtures under ``tests/golden/``; ``tests/test_oracle_golden.py`` checks this
file against them) and the motor model additionally against the reference's only
in-repo known-answer file (sim2real/motorid_utilities/sample_sim_euler_integration.csv,
first rows committed in ``tests/golden/motor_euler_csv.json``).

PARITY UNPINNED: ``rigid_body_integrate`` (reference row a13).  The reference
delegates integration to Isaac Gym / PhysX (``gym.simulate``,
env_manager/IGE_env_manager.py:477), a closed binary that is not in the tree
and not installable here.  The integrator below is *our written specification*
(DESIGN.md section "Integrator spec"), following only call-site facts: forces
and torques are per-link, link-local (IGE_env_manager.py:444-449); state layout
[x y z qx qy qz qw vx vy vz wx wy wz] with world-frame velocities
(IGE_env_manager.py:347-358); dt / gravity from config/sim_config/base_sim_config.py:20-22;
linear/angular damping and velocity caps from config/robot_config/base_quad_config.py:93-97.

``matrix_to_quaternion`` is pytorch3d's (not in the tree, unpinned version):
restated from its published algorithm; the sign of the result is immaterial
downstream (quat_to_rotation_matrix and quat_rotate are even in q).

All functions are dtype-parametric: fp32 reproduces the reference's arithmetic
order, fp64 is used as "truth" when a test needs to apportion error.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, Optional

import numpy as np
import torch

PI = math.pi

# controller ids shared with include/aerial_gym_b200.h (AGX_CTRL_*)
CTRL_NONE = 0
CTRL_ATTITUDE = 1
CTRL_POSITION = 2
CTRL_VELOCITY = 3
CTRL_ACCELERATION = 4
CTRL_RATES = 5
CTRL_FULLY_ACTUATED = 6
CTRL_VELOCITY_STEERING = 7


# --------------------------------------------------------------------------------------
# quaternion / rotation helpers (xyzw convention)        reference: utils/math.py
# --------------------------------------------------------------------------------------
def quat_rotate(q, v):
    """utils/math.py:58-65 -- v*(2w^2-1) + 2w (q_v x v) + 2 q_v (q_v . v)."""
    qw = q[:, 3:4]
    qv = q[:, :3]
    a = v * (2.0 * qw * qw - 1.0)
    b = torch.cross(qv, v, dim=-1) * qw * 2.0
    c = qv * (qv * v).sum(-1, keepdim=True) * 2.0
    return a + b + c


def quat_rotate_inverse(q, v):
    """utils/math.py:339-347 -- same with the cross term negated."""
    qw = q[:, 3:4]
    qv = q[:, :3]
    a = v * (2.0 * qw * qw - 1.0)
    b = torch.cross(qv, v, dim=-1) * qw * 2.0
    c = qv * (qv * v).sum(-1, keepdim=True) * 2.0
    return a - b + c


def quat_apply(q, v):
    """utils/math.py:313-320."""
    xyz = q[:, :3]
    t = torch.cross(xyz, v, dim=-1) * 2
    return v + q[:, 3:4] * t + torch.cross(xyz, t, dim=-1)


def quat_conjugate(q):
    return torch.cat((-q[:, :3], q[:, 3:4]), dim=-1)


def quat_mul(a, b):
    """utils/math.py:242-263 (the 9-multiply form, same association order)."""
    x1, y1, z1, w1 = a[:, 0], a[:, 1], a[:, 2], a[:, 3]
    x2, y2, z2, w2 = b[:, 0], b[:, 1], b[:, 2], b[:, 3]
    ww = (z1 + x1) * (x2 + y2)
    yy = (w1 - y1) * (w2 + z2)
    zz = (w1 + y1) * (w2 - z2)
    xx = ww + yy + zz
    qq = 0.5 * (xx + (z1 - x1) * (x2 - y2))
    w = qq - ww + (z1 - y1) * (y2 - z2)
    x = qq - xx + (x1 + w1) * (x2 + w2)
    y = qq - yy + (w1 - x1) * (y2 + z2)
    z = qq - zz + (z1 + y1) * (w2 - x2)
    return torch.stack([x, y, z, w], dim=-1)


def quat_to_rotation_matrix(q):
    """utils/math.py:266-293 -> [N,3,3] row-major."""
    x, y, z, w = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    xx, xy, xz, xw = x * x, x * y, x * z, x * w
    yy, yz, yw = y * y, y * z, y * w
    zz, zw = z * z, z * w
    m = torch.stack(
        [
            1 - 2.0 * (yy + zz), 2.0 * (xy - zw), 2.0 * (xz + yw),
            2.0 * (xy + zw), 1 - 2.0 * (xx + zz), 2.0 * (yz - xw),
            2.0 * (xz - yw), 2.0 * (yz + xw), 1 - 2.0 * (xx + yy),
        ],
        dim=-1,
    )
    return m.view(-1, 3, 3)


def euler_xyz_from_quat(q):
    """utils/math.py:123-146 (get_euler_xyz_tensor): each angle wrapped to [0, 2pi)."""
    qx, qy, qz, qw = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    sinr_cosp = 2.0 * (qw * qx + qy * qz)
    cosr_cosp = qw * qw - qx * qx - qy * qy + qz * qz
    roll = torch.atan2(sinr_cosp, cosr_cosp)
    sinp = 2.0 * (qw * qy - qz * qx)
    half_pi = torch.full_like(sinp, PI / 2.0)
    pitch = torch.where(torch.abs(sinp) >= 1, half_pi * torch.sign(sinp), torch.asin(sinp))
    siny_cosp = 2.0 * (qw * qz + qx * qy)
    cosy_cosp = qw * qw + qx * qx - qy * qy - qz * qz
    yaw = torch.atan2(siny_cosp, cosy_cosp)
    return torch.stack([roll % (2 * PI), pitch % (2 * PI), yaw % (2 * PI)], dim=-1)


def ssa(a):
    """utils/math.py:149-152 smallest signed angle."""
    return torch.remainder(a + PI, 2 * PI) - PI


def quat_from_euler_xyz(roll, pitch, yaw):
    """utils/math.py:155-172 / 183-197."""
    cy, sy = torch.cos(yaw * 0.5), torch.sin(yaw * 0.5)
    cr, sr = torch.cos(roll * 0.5), torch.sin(roll * 0.5)
    cp, sp = torch.cos(pitch * 0.5), torch.sin(pitch * 0.5)
    qw = cy * cr * cp + sy * sr * sp
    qx = cy * sr * cp - sy * cr * sp
    qy = cy * cr * sp + sy * sr * cp
    qz = sy * cr * cp - cy * sr * sp
    return torch.stack([qx, qy, qz, qw], dim=-1)


def vehicle_frame_quat_from_quat(q):
    """utils/math.py:175-180: keep only the (wrapped, [0,2pi)) yaw."""
    e = euler_xyz_from_quat(q)
    zero = torch.zeros_like(e[:, 0])
    return quat_from_euler_xyz(zero, zero, e[:, 2])


def matrix_to_quaternion_xyzw(R):
    """pytorch3d.transforms.matrix_to_quaternion (published algorithm), reordered to xyzw
    as base_lee_controller.py:188-189 does."""
    m00, m01, m02 = R[:, 0, 0], R[:, 0, 1], R[:, 0, 2]
    m10, m11, m12 = R[:, 1, 0], R[:, 1, 1], R[:, 1, 2]
    m20, m21, m22 = R[:, 2, 0], R[:, 2, 1], R[:, 2, 2]
    t = torch.stack(
        [1.0 + m00 + m11 + m22, 1.0 + m00 - m11 - m22, 1.0 - m00 + m11 - m22, 1.0 - m00 - m11 + m22],
        dim=-1,
    )
    q_abs = torch.sqrt(torch.clamp(t, min=0.0))
    cand = torch.stack(
        [
            torch.stack([q_abs[:, 0] ** 2, m21 - m12, m02 - m20, m10 - m01], dim=-1),
            torch.stack([m21 - m12, q_abs[:, 1] ** 2, m10 + m01, m02 + m20], dim=-1),
            torch.stack([m02 - m20, m10 + m01, q_abs[:, 2] ** 2, m12 + m21], dim=-1),
            torch.stack([m10 - m01, m20 + m02, m21 + m12, q_abs[:, 3] ** 2], dim=-1),
        ],
        dim=-2,
    )
    cand = cand / (2.0 * torch.clamp(q_abs, min=0.1)[..., None])
    idx = q_abs.argmax(dim=-1)
    wxyz = cand[torch.arange(R.shape[0]), idx]
    return torch.stack([wxyz[:, 1], wxyz[:, 2], wxyz[:, 3], wxyz[:, 0]], dim=-1)


# --------------------------------------------------------------------------------------
# model description
# --------------------------------------------------------------------------------------
@dataclass
class Hp1Model:
    """Static (per robot x controller) description; plain Python numbers / numpy arrays."""

    num_motors: int = 4
    controller: int = CTRL_ATTITUDE
    dt: float = 0.01
    gravity: tuple = (0.0, 0.0, -9.81)
    mass: float = 0.25
    inertia: np.ndarray = field(default_factory=lambda: np.diag([8.45e-4, 8.45e-4, 1.69e-3]))
    com: np.ndarray = field(default_factory=lambda: np.zeros(3))
    # control allocation (control_allocation.py)
    allocation_matrix: np.ndarray = None  # [6, M]
    motor_directions: np.ndarray = None  # [M]
    thrust_to_torque_ratio: float = 0.01
    force_application_level: str = "motor_link"
    link_r: np.ndarray = None  # [M,3] motor link origins in base frame (URDF joints)
    link_R: np.ndarray = None  # [M,3,3] motor link orientation in base frame
    # motor model (motor_model.py)
    use_rps: bool = True
    integration_scheme: str = "rk4"
    use_discrete_approximation: bool = True
    min_thrust: float = 0.0
    max_thrust: float = 2.0
    max_thrust_rate: float = 100000.0
    # ranges used on reset
    tau_inc_range: tuple = (0.04, 0.04)
    tau_dec_range: tuple = (0.04, 0.04)
    k_thrust_range: tuple = (0.00000926312, 0.00001826312)
    # controller (lee_controller_config.py)
    max_yaw_rate: float = PI / 3.0
    K_pos_range: tuple = ((2.0, 2.0, 1.0), (3.0, 3.0, 2.0))
    K_vel_range: tuple = ((2.0, 2.0, 2.0), (3.0, 3.0, 3.0))
    K_rot_range: tuple = ((0.8, 0.8, 0.4), (1.2, 1.2, 0.6))
    K_angvel_range: tuple = ((0.1, 0.1, 0.1), (0.2, 0.2, 0.2))
    randomize_params: bool = False
    # drag (base_multirotor.py:260-285)
    drag_lin1: tuple = (0.0, 0.0, 0.0)
    drag_lin2: tuple = (0.0, 0.0, 0.0)
    drag_ang1: tuple = (0.0, 0.0, 0.0)
    drag_ang2: tuple = (0.0, 0.0, 0.0)
    # disturbance (base_multirotor.py:213-234)
    enable_disturbance: bool = False
    prob_apply_disturbance: float = 0.02
    max_disturbance: tuple = (0.75, 0.75, 0.75, 0.004, 0.004, 0.004)
    # integrator spec (ours; PhysX-style) -- base_quad_config.py:93-97
    linear_damping: float = 0.01
    angular_damping: float = 0.01
    max_linear_velocity: float = 100.0
    max_angular_velocity: float = 100.0
    gyroscopic: bool = True
    # reset (base_quad_config.py:30-59, empty_env.py:27-31)
    min_init_state: tuple = (0.1, 0.15, 0.15, 0, 0, -PI / 6, 1.0, -0.2, -0.2, -0.2, -0.2, -0.2, -0.2)
    max_init_state: tuple = (0.2, 0.85, 0.85, 0, 0, PI / 6, 1.0, 0.2, 0.2, 0.2, 0.2, 0.2, 0.2)
    bounds_lower_range: tuple = ((-1.0, -1.0, -1.0), (-1.0, -1.0, -1.0))
    bounds_upper_range: tuple = ((1.0, 1.0, 1.0), (1.0, 1.0, 1.0))

    def __post_init__(self):
        M = self.num_motors
        if self.allocation_matrix is None:
            self.allocation_matrix = np.array(
                [
                    [0.0, 0.0, 0.0, 0.0],
                    [0.0, 0.0, 0.0, 0.0],
                    [1.0, 1.0, 1.0, 1.0],
                    [-0.13, -0.13, 0.13, 0.13],
                    [-0.13, 0.13, 0.13, -0.13],
                    [-0.01, 0.01, -0.01, 0.01],
                ]
            )
        if self.motor_directions is None:
            self.motor_directions = np.array([1, -1, 1, -1], dtype=np.float64)
        if self.link_r is None:
            # resources/robots/quad/quad.urdf joints base_link_to_motor_{0..3}
            self.link_r = np.array(
                [[0.13, -0.13, 0.0], [-0.13, -0.13, 0.0], [-0.13, 0.13, 0.0], [0.13, 0.13, 0.0]]
            )
        if self.link_R is None:
            self.link_R = np.tile(np.eye(3), (M, 1, 1))
        self.allocation_matrix = np.asarray(self.allocation_matrix, dtype=np.float64)
        self.motor_directions = np.asarray(self.motor_directions, dtype=np.float64)
        self.link_r = np.asarray(self.link_r, dtype=np.float64)
        self.link_R = np.asarray(self.link_R, dtype=np.float64)
        self.inertia = np.asarray(self.inertia, dtype=np.float64)
        self.com = np.asarray(self.com, dtype=np.float64)

    # ---- derived constants -----------------------------------------------------------
    def pinv_allocation(self, dtype=torch.float32):
        """control_allocation.py:46-48: torch.linalg.pinv of the fp32 matrix."""
        A = torch.tensor(self.allocation_matrix, dtype=torch.float32)
        return torch.linalg.pinv(A).to(dtype)

    def wrench_map(self):
        """[6,M] map motor thrust -> base-frame wrench about the COM.

        motor_link: column i = [R_i e_z ; (r_i-c) x R_i e_z - cq*dir_i*R_i e_z]
        (control_allocation.py:103-114 applied LOCAL_SPACE at link i, IGE_env_manager.py:444-449;
        SURVEY Appendix B).  Any other level: the allocation matrix itself, applied to body 0
        (control_allocation.py:60-63, base_multirotor.py:152-159)."""
        M = self.num_motors
        if self.force_application_level == "motor_link":
            W = np.zeros((6, M))
            for i in range(M):
                ez = self.link_R[i] @ np.array([0.0, 0.0, 1.0])
                W[0:3, i] = ez
                W[3:6, i] = np.cross(self.link_r[i] - self.com, ez) - (
                    self.thrust_to_torque_ratio * self.motor_directions[i] * ez
                )
            return W
        W = self.allocation_matrix.copy()
        # wrench given at base-link origin; move the torque reference to the COM
        for i in range(M):
            W[3:6, i] += np.cross(-self.com, W[0:3, i])
        return W


@dataclass
class Hp1State:
    """Per-env tensors (all leading dim N).  ``root`` is the [N,13] robot state."""

    root: torch.Tensor
    thrust: torch.Tensor  # [N,M] current motor thrust (motor_model.current_motor_thrust)
    tau_inc: torch.Tensor  # [N,M]
    tau_dec: torch.Tensor  # [N,M]
    k_thrust: torch.Tensor  # [N,M]
    K_pos: torch.Tensor  # [N,3]
    K_vel: torch.Tensor
    K_rot: torch.Tensor
    K_angvel: torch.Tensor
    bounds_min: torch.Tensor  # [N,3]
    bounds_max: torch.Tensor
    sim_steps: torch.Tensor  # int32 [N]
    derived: Dict[str, torch.Tensor] = field(default_factory=dict)

    def clone(self):
        return Hp1State(
            **{
                k: (v.clone() if torch.is_tensor(v) else {kk: vv.clone() for kk, vv in v.items()})
                for k, v in self.__dict__.items()
            }
        )


def make_state(model: Hp1Model, N: int, dtype=torch.float32) -> Hp1State:
    """Allocate a state with the reference's construction-time defaults: gains at the
    mid-point of min/max (base_lee_controller.py:59-62)."""
    M = model.num_motors

    def mid(rng):
        lo, hi = torch.tensor(rng[0], dtype=dtype), torch.tensor(rng[1], dtype=dtype)
        return ((hi + lo) / 2.0).expand(N, -1).clone()

    z = lambda *s: torch.zeros(*s, dtype=dtype)
    root = z(N, 13)
    root[:, 6] = 1.0
    return Hp1State(
        root=root,
        thrust=z(N, M),
        tau_inc=torch.full((N, M), model.tau_inc_range[0], dtype=dtype),
        tau_dec=torch.full((N, M), model.tau_dec_range[0], dtype=dtype),
        k_thrust=torch.full((N, M), model.k_thrust_range[0], dtype=dtype),
        K_pos=mid(model.K_pos_range),
        K_vel=mid(model.K_vel_range),
        K_rot=mid(model.K_rot_range),
        K_angvel=mid(model.K_angvel_range),
        bounds_min=torch.tensor(model.bounds_lower_range[0], dtype=dtype).expand(N, -1).clone(),
        bounds_max=torch.tensor(model.bounds_upper_range[0], dtype=dtype).expand(N, -1).clone(),
        sim_steps=torch.zeros(N, dtype=torch.int32),
    )


# --------------------------------------------------------------------------------------
# a1  update_states                       robots/base_multirotor.py:287-294
# --------------------------------------------------------------------------------------
def update_states(root):
    q = root[:, 3:7]
    v = root[:, 7:10]
    w = root[:, 10:13]
    euler = ssa(euler_xyz_from_quat(q))
    q_veh = vehicle_frame_quat_from_quat(q)
    return {
        "euler": euler,
        "vehicle_orientation": q_veh,
        "vehicle_linvel": quat_rotate_inverse(q_veh, v),
        "body_linvel": quat_rotate_inverse(q, v),
        "body_angvel": quat_rotate_inverse(q, w),
    }


# --------------------------------------------------------------------------------------
# a2-a7  Lee controllers                  control/controllers/*.py
# --------------------------------------------------------------------------------------
def _compute_acceleration(st: Hp1State, d, sp_pos, sp_vel):
    """base_lee_controller.py:120-134."""
    pos_err = sp_pos - st.root[:, 0:3]
    sp_vel_world = quat_rotate(d["vehicle_orientation"], sp_vel)
    vel_err = sp_vel_world - st.root[:, 7:10]
    return st.K_pos * pos_err + st.K_vel * vel_err


def _euler_rates_to_body_rates(euler, rates):
    """base_lee_controller.py:200-215.  The reference builds T in a shared [N,3,3] scratch
    that is zero (or holds stale entries that multiply the zero roll/pitch rates); only the
    entries written there are restated: T = [[1,0,-sp],[0,cr,sr*cp],[0,-sr,cr*cp]]."""
    s_p, c_p = torch.sin(euler[:, 1]), torch.cos(euler[:, 1])
    s_r, c_r = torch.sin(euler[:, 0]), torch.cos(euler[:, 0])
    zero = torch.zeros_like(s_p)
    one = torch.ones_like(s_p)
    T = torch.stack(
        [one, zero, -s_p, zero, c_r, s_r * c_p, zero, -s_r, c_r * c_p], dim=-1
    ).view(-1, 3, 3)
    return torch.bmm(T, rates.unsqueeze(2)).squeeze(2)


def _compute_body_torque(model: Hp1Model, st: Hp1State, d, q_des, w_des, J):
    """base_lee_controller.py:136-154.  Returns (torque, clamped w_des)."""
    w_des = w_des.clone()
    w_des[:, 2] = torch.clamp(w_des[:, 2], -model.max_yaw_rate, model.max_yaw_rate)
    q = st.root[:, 3:7]
    q_err = quat_mul(quat_conjugate(q), q_des)
    R_err = quat_to_rotation_matrix(q_err)
    S = torch.transpose(R_err, -2, -1) - R_err
    rot_err = 0.5 * torch.stack([-S[:, 1, 2], S[:, 0, 2], -S[:, 0, 1]], dim=1)  # math.py:34-42
    W = d["body_angvel"]
    angvel_err = W - quat_rotate(q_err, w_des)
    JW = torch.bmm(J, W.unsqueeze(2)).squeeze(2)
    ff = torch.cross(W, JW, dim=1)
    return -st.K_rot * rot_err - st.K_angvel * angvel_err + ff


def _desired_orientation_pos_vel(forces, yaw):
    """base_lee_controller.py:173-194 (b3 from force, b2 = b3 x c1, b1 = b2 x b3)."""
    b3 = forces / torch.norm(forces, dim=1, keepdim=True)
    c1 = torch.zeros_like(forces)
    c1[:, 0] = torch.cos(yaw)
    c1[:, 1] = torch.sin(yaw)
    b2 = torch.cross(b3, c1, dim=1)
    b2 = b2 / torch.norm(b2, dim=1, keepdim=True)
    b1 = torch.cross(b2, b3, dim=1)
    R = torch.stack([b1, b2, b3], dim=2)  # columns
    return matrix_to_quaternion_xyzw(R)


def _desired_orientation_forces_yaw(forces, yaw):
    """base_lee_controller.py:157-169."""
    c_phi_s_theta = forces[:, 0]
    s_phi = -forces[:, 1]
    c_phi_c_theta = forces[:, 2]
    pitch = torch.atan2(c_phi_s_theta, c_phi_c_theta)
    roll = torch.atan2(s_phi, torch.sqrt(c_phi_c_theta**2 + c_phi_s_theta**2))
    return quat_from_euler_xyz(roll, pitch, yaw)


def controller_wrench(model: Hp1Model, st: Hp1State, d, actions):
    """Dispatch on controller id; returns the [N,6] wrench command (or the pass-through
    motor command for CTRL_NONE, no_control.py:29-30).  ``actions`` already clamped to +-10
    (base_multirotor.py:207-211)."""
    N = actions.shape[0]
    dt_ = actions.dtype
    g = torch.tensor(model.gravity, dtype=dt_).expand(N, -1)
    m = torch.full((N, 1), model.mass, dtype=dt_)
    J = torch.tensor(model.inertia, dtype=dt_).expand(N, -1, -1)
    wrench = torch.zeros(N, 6, dtype=dt_)
    c = model.controller
    euler = d["euler"]
    zeros3 = torch.zeros(N, 3, dtype=dt_)
    if c == CTRL_NONE:
        return actions
    if c == CTRL_ATTITUDE:  # attitude_control.py:16-43
        wrench[:, 2] = (actions[:, 0] + 1.0) * m.squeeze(1) * torch.norm(g, dim=1)
        rates = zeros3.clone()
        rates[:, 2] = actions[:, 3]
        w_des = _euler_rates_to_body_rates(euler, rates)
        q_des = quat_from_euler_xyz(actions[:, 1], actions[:, 2], euler[:, 2])
        wrench[:, 3:6] = _compute_body_torque(model, st, d, q_des, w_des, J)
        return wrench
    if c == CTRL_RATES:
        # rates_control.py:23-26.  The reference line `(a0 - gravity) * mass` mixes [N] with
        # [N,3] and raises for every N != 1; this restates the evident intent
        # (thrust = (a0 - g_z) * m) and is NOT parity-checkable against the reference.
        wrench[:, 2] = (actions[:, 0] - g[:, 2]) * m.squeeze(1)
        wrench[:, 3:6] = _compute_body_torque(model, st, d, st.root[:, 3:7], actions[:, 1:4], J)
        return wrench
    if c == CTRL_FULLY_ACTUATED:  # fully_actuated_control.py:14-32
        qn = actions[:, 3:7]
        qn = qn / torch.clamp(torch.norm(qn, dim=-1, keepdim=True), min=1e-9)
        accel = _compute_acceleration(st, d, actions[:, 0:3], zeros3)
        forces = m * (accel - g)
        wrench[:, 0:3] = quat_rotate_inverse(st.root[:, 3:7], forces)
        wrench[:, 3:6] = _compute_body_torque(model, st, d, qn, zeros3, J)
        return wrench
    # thrust-vectoring family
    if c == CTRL_POSITION:  # position_control.py:16-51
        accel = _compute_acceleration(st, d, actions[:, 0:3], zeros3)
        forces = (accel - g) * m
    elif c in (CTRL_VELOCITY, CTRL_VELOCITY_STEERING):  # velocity_control.py:17-53
        accel = _compute_acceleration(st, d, st.root[:, 0:3], actions[:, 0:3])
        forces = (accel - g) * m
    elif c == CTRL_ACCELERATION:  # acceleration_control.py:16-46
        accel = actions[:, 0:3]
        forces = m * (accel - g)
    else:
        raise ValueError(f"unknown controller id {c}")
    Rz = quat_to_rotation_matrix(st.root[:, 3:7])[:, :, 2]
    wrench[:, 2] = torch.sum(forces * Rz, dim=1)
    if c == CTRL_POSITION:
        q_des = _desired_orientation_pos_vel(forces, actions[:, 3])
        w_des = zeros3
    elif c == CTRL_VELOCITY:
        q_des = _desired_orientation_pos_vel(forces, euler[:, 2])
        rates = zeros3.clone()
        rates[:, 2] = actions[:, 3]
        w_des = _euler_rates_to_body_rates(euler, rates)
    elif c == CTRL_VELOCITY_STEERING:  # velocity_steeing_angle_controller.py:16-50
        q_des = _desired_orientation_pos_vel(forces, actions[:, 3])
        w_des = zeros3
    else:  # acceleration
        q_des = _desired_orientation_forces_yaw(forces, euler[:, 2])
        rates = zeros3.clone()
        rates[:, 2] = actions[:, 3]
        w_des = _euler_rates_to_body_rates(euler, rates)
    wrench[:, 3:6] = _compute_body_torque(model, st, d, q_des, w_des, J)
    return wrench


# --------------------------------------------------------------------------------------
# a9  motor model                         control/motor_model.py:88-251
# --------------------------------------------------------------------------------------
def _rate(err, mix, max_rate):
    return torch.clamp(mix * err, -max_rate, max_rate)  # motor_model.py:160-162


def _rk4(ref, cur, mix, max_rate, dt):
    """motor_model.py:165-199."""
    k1 = _rate(ref - cur, mix, max_rate)
    k2 = _rate(ref - (cur + 0.5 * dt * k1), mix, max_rate)
    k3 = _rate(ref - (cur + 0.5 * dt * k2), mix, max_rate)
    k4 = _rate(ref - (cur + dt * k3), mix, max_rate)
    return (dt / 6.0) * (k1 + 2.0 * k2 + 2.0 * k3 + k4)


def motor_update(model: Hp1Model, st: Hp1State, ref_thrust):
    """MotorModel.update_motor_thrusts; returns the new thrust [N,M] (caller stores it)."""
    dt = model.dt
    ref = torch.clamp(ref_thrust, model.min_thrust, model.max_thrust)
    cur = st.thrust
    err = ref - cur
    tau = torch.where(torch.sign(cur) * torch.sign(err) < 0, st.tau_dec, st.tau_inc)
    mix = 1.0 / (dt + tau) if model.use_discrete_approximation else 1.0 / tau
    rk4 = model.integration_scheme != "euler"  # default rk4, motor_model.py:13-19
    if model.use_rps:
        k = st.k_thrust
        rpm = torch.sqrt(cur / k)
        rpm_ref = torch.sqrt(ref / k)
        if rk4:
            rpm = rpm + _rk4(rpm_ref, rpm, mix, model.max_thrust_rate, dt)
        else:
            rpm = rpm + _rate(rpm_ref - rpm, mix, model.max_thrust_rate) * dt
        return k * rpm**2
    if rk4:
        return cur + _rk4(ref, cur, mix, model.max_thrust_rate, dt)
    return cur + _rate(err, mix, model.max_thrust_rate) * dt


# --------------------------------------------------------------------------------------
# a8/a10/a11  allocation -> per-link force/torque tensors
# --------------------------------------------------------------------------------------
def allocate(model: Hp1Model, st: Hp1State, command):
    """ControlAllocator.allocate_output (control_allocation.py:52-65).

    Returns (new_thrust [N,M], forces [N,L,3], torques [N,L,3]) where L = M link-local
    entries for motor_link mode and L = 1 (body 0) otherwise."""
    dt_ = command.dtype
    N = command.shape[0]
    if model.controller == CTRL_NONE:
        ref = command  # update_motor_thrusts_with_forces
    else:
        Apinv = model.pinv_allocation(dt_).expand(N, -1, -1)
        ref = torch.bmm(Apinv, command.unsqueeze(-1)).squeeze(-1)
    f = motor_update(model, st, ref)
    if model.force_application_level == "motor_link":
        z = torch.zeros_like(f)
        forces = torch.stack([z, z, f], dim=2)
        dirs = torch.tensor(model.motor_directions, dtype=dt_)
        torques = model.thrust_to_torque_ratio * forces * (-dirs[None, :, None])
        return f, forces, torques
    A = torch.tensor(model.allocation_matrix, dtype=torch.float32).to(dt_).expand(N, -1, -1)
    w = torch.bmm(A, f.unsqueeze(-1)).squeeze(-1)
    return f, w[:, 0:3].unsqueeze(1), w[:, 3:6].unsqueeze(1)


def drag_wrench(model: Hp1Model, d):
    """simulate_drag (base_multirotor.py:260-285): added to body 0, body frame."""
    vb, wb = d["body_linvel"], d["body_angvel"]
    dt_ = vb.dtype
    k1 = torch.tensor(model.drag_lin1, dtype=dt_)
    k2 = torch.tensor(model.drag_lin2, dtype=dt_)
    a1 = torch.tensor(model.drag_ang1, dtype=dt_)
    a2 = torch.tensor(model.drag_ang2, dtype=dt_)
    f = (-k1 * vb) + (-k2 * torch.norm(vb, dim=-1).unsqueeze(-1) * vb)
    t = (-a1 * wb) + (-a2 * wb.abs() * wb)
    return f, t


def draw_disturbance(model: Hp1Model, N: int, dtype=torch.float32, generator=None):
    """apply_disturbance (base_multirotor.py:213-234) in the reference's RNG call order:
    bernoulli(p*ones(N)) -> rand_like [N,3] (force) -> rand_like [N,3] (torque).
    Returns the gated body-0 wrench [N,6] or None when disabled."""
    if not model.enable_disturbance:
        return None
    occ = torch.bernoulli(model.prob_apply_disturbance * torch.ones(N, dtype=dtype), generator=generator)
    mx = torch.tensor(model.max_disturbance, dtype=dtype).expand(N, -1)
    u1 = torch.rand(N, 3, dtype=dtype, generator=generator)
    u2 = torch.rand(N, 3, dtype=dtype, generator=generator)
    f = ((mx[:, 0:3] - (-mx[:, 0:3])) * u1 + (-mx[:, 0:3])) * occ.unsqueeze(1)
    t = ((mx[:, 3:6] - (-mx[:, 3:6])) * u2 + (-mx[:, 3:6])) * occ.unsqueeze(1)
    return torch.cat([f, t], dim=1)


def link_wrenches_to_body(model: Hp1Model, forces, torques, body0_force, body0_torque):
    """Reduce link-local forces/torques to one base-frame wrench about the COM
    (SURVEY Appendix B): F = sum R_i F_i ; tau = sum (r_i - c) x R_i F_i + R_i T_i.
    Body 0 (base link, r = 0, R = I) carries drag and disturbance."""
    dt_ = forces.dtype
    com = torch.tensor(model.com, dtype=dt_)
    if model.force_application_level == "motor_link":
        R = torch.tensor(model.link_R, dtype=dt_)  # [M,3,3]
        r = torch.tensor(model.link_r, dtype=dt_)  # [M,3]
        Fb = torch.einsum("mij,nmj->nmi", R, forces)
        Tb = torch.einsum("mij,nmj->nmi", R, torques)
        F = Fb.sum(1)
        T = (torch.cross((r - com)[None].expand_as(Fb), Fb, dim=-1) + Tb).sum(1)
    else:
        F = forces[:, 0]
        T = torques[:, 0] + torch.cross((-com).expand_as(F), F, dim=-1)
    F = F + body0_force
    T = T + body0_torque + torch.cross((-com).expand_as(body0_force), body0_force, dim=-1)
    return F, T


# --------------------------------------------------------------------------------------
# a13  rigid-body integrator -- OUR SPEC (parity unpinned, see module docstring)
# --------------------------------------------------------------------------------------
def rigid_body_integrate(model: Hp1Model, root, F_body, T_body):
    """Semi-implicit Euler, PhysX-style damping and velocity caps.

      a      = R(q) F_b / m + g
      v'     = (v + dt a) * max(0, 1 - dt*lin_damp);  |v'| capped at max_linear_velocity
      W      = R(q)^T w            (body rates)
      W'     = W + dt J^-1 (T_b - W x J W)            (gyroscopic term if model.gyroscopic)
      w'     = (R(q) W') * max(0, 1 - dt*ang_damp);   |w'| capped at max_angular_velocity
      x'     = x + dt v'
      q'     = normalize( dq (x) q ),  dq = [w'/|w'| sin(|w'|dt/2), cos(|w'|dt/2)]  (world-frame, left)
    """
    dt_ = root.dtype
    dt = model.dt
    x, q, v, w = root[:, 0:3], root[:, 3:7], root[:, 7:10], root[:, 10:13]
    g = torch.tensor(model.gravity, dtype=dt_)
    J = torch.tensor(model.inertia, dtype=dt_)
    Jinv = torch.tensor(np.linalg.inv(model.inertia), dtype=dt_)
    a = quat_rotate(q, F_body) / model.mass + g
    v_new = (v + dt * a) * max(0.0, 1.0 - dt * model.linear_damping)
    vn = torch.norm(v_new, dim=1, keepdim=True)
    v_new = torch.where(vn > model.max_linear_velocity, v_new * (model.max_linear_velocity / vn), v_new)
    W = quat_rotate_inverse(q, w)
    JW = W @ J.T
    rhs = T_body - torch.cross(W, JW, dim=1) if model.gyroscopic else T_body
    W_new = W + dt * (rhs @ Jinv.T)
    w_new = quat_rotate(q, W_new) * max(0.0, 1.0 - dt * model.angular_damping)
    wn = torch.norm(w_new, dim=1, keepdim=True)
    w_new = torch.where(wn > model.max_angular_velocity, w_new * (model.max_angular_velocity / wn), w_new)
    x_new = x + dt * v_new
    wn = torch.norm(w_new, dim=1, keepdim=True)
    half = 0.5 * dt * wn
    s_over = torch.where(wn > 0, torch.sin(half) / torch.where(wn > 0, wn, torch.ones_like(wn)), torch.zeros_like(wn))
    dq = torch.cat([w_new * s_over, torch.cos(half)], dim=1)
    q_new = quat_mul(dq, q)
    q_new = q_new / torch.norm(q_new, dim=1, keepdim=True)
    return torch.cat([x_new, q_new, v_new, w_new], dim=1)


# --------------------------------------------------------------------------------------
# one physics step = BaseMultirotor.step + integrator
# --------------------------------------------------------------------------------------
def physics_step(model: Hp1Model, st: Hp1State, actions, disturbance=None):
    """robots/base_multirotor.py:296-307 then the integrator.  Mutates ``st`` in place
    (root, thrust, derived = the PRE-physics derived states, i.e. stale afterwards, exactly
    like the reference -- SURVEY 3.1).  ``disturbance``: optional [N,6] body-0 wrench already
    gated by the Bernoulli mask (the draws themselves stay in torch, in reference order).
    Returns dict with the intermediate quantities tests compare."""
    d = update_states(st.root)
    a = torch.clamp(actions, -10.0, 10.0)
    cmd = controller_wrench(model, st, d, a)
    f_new, forces, torques = allocate(model, st, cmd)
    st.thrust = f_new
    df, dtq = drag_wrench(model, d)
    if disturbance is not None:
        df = df + disturbance[:, 0:3]
        dtq = dtq + disturbance[:, 3:6]
    F, T = link_wrenches_to_body(model, forces, torques, df, dtq)
    st.root = rigid_body_integrate(model, st.root, F, T)
    st.derived = d
    return {"wrench_cmd": cmd, "link_forces": forces, "link_torques": torques, "F_body": F, "T_body": T}


# --------------------------------------------------------------------------------------
# a16  position task epilogue             task/position_setpoint_task/position_setpoint_task.py
# --------------------------------------------------------------------------------------
def position_task_reward(st: Hp1State, target, crashes):
    """compute_rewards_and_crashes + compute_reward (:205-282).  Uses the STALE vehicle
    orientation / body angvel in st.derived.  Returns (reward [N], crashes bool [N])."""
    d = st.derived
    pos = st.root[:, 0:3]
    q = st.root[:, 3:7]
    e = quat_apply(quat_conjugate(d["vehicle_orientation"]), target - pos)
    dist = torch.norm(e, dim=1)
    pos_reward = 3.0 * torch.exp(-8.0 * dist * dist) + 2.0 * torch.exp(-4.0 * dist * dist)
    dist_reward = (20 - dist) / 40.0
    ez = torch.zeros_like(pos)
    ez[:, 2] = 1
    ups = quat_rotate(q, ez)
    tilt = torch.abs(1 - ups[:, 2])
    up_reward = 0.2 / (0.1 + tilt * tilt)
    spin = torch.norm(d["body_angvel"], dim=1)
    ang_reward = (1.0 / (1.0 + spin * spin)) * 3
    total = pos_reward + dist_reward + pos_reward * (up_reward + ang_reward)
    crashes = torch.where(dist > 8.0, torch.ones_like(crashes), crashes)
    total = torch.where(crashes, -20 * torch.ones_like(total), total)
    return total, crashes


def position_task_obs(st: Hp1State, target):
    """process_obs_for_task (:194-203)."""
    d = st.derived
    return torch.cat([target - st.root[:, 0:3], st.root[:, 3:7], d["body_linvel"], d["body_angvel"]], dim=1)


# --------------------------------------------------------------------------------------
# a15  reset                              (draws are explicit uniforms in [0,1))
# --------------------------------------------------------------------------------------
@dataclass
class ResetDraws:
    """Uniform [0,1) draws in the reference's call order (SURVEY 3.1):
    IGE bounds lower/upper [N,3]x2 -> robot state [N,13] -> gains 4x[N,3] (only consumed if
    randomize_params) -> motor tau_inc, tau_dec, thrust [N,M] -> k_thrust [N,M] (if use_rps)."""

    bounds_lo: torch.Tensor
    bounds_hi: torch.Tensor
    state: torch.Tensor
    K_pos: Optional[torch.Tensor]
    K_vel: Optional[torch.Tensor]
    K_rot: Optional[torch.Tensor]
    K_angvel: Optional[torch.Tensor]
    tau_inc: torch.Tensor
    tau_dec: torch.Tensor
    thrust: torch.Tensor
    k_thrust: Optional[torch.Tensor]


def draw_reset_uniforms(model: Hp1Model, N: int, dtype=torch.float32, generator=None) -> ResetDraws:
    r = lambda *s: torch.rand(*s, dtype=dtype, generator=generator)
    M = model.num_motors
    bl, bh, s = r(N, 3), r(N, 3), r(N, 13)
    if model.randomize_params:
        kp, kv, kr, kw = r(N, 3), r(N, 3), r(N, 3), r(N, 3)
    else:
        kp = kv = kr = kw = None
    ti, td, th = r(N, M), r(N, M), r(N, M)
    kt = r(N, M) if model.use_rps else None
    return ResetDraws(bl, bh, s, kp, kv, kr, kw, ti, td, th, kt)


def _lerp_rand(lo, hi, u):
    """torch_rand_float_tensor (utils/math.py:51-54): (upper - lower) * u + lower."""
    return (hi - lo) * u + lo


def reset_envs(model: Hp1Model, st: Hp1State, mask, draws: ResetDraws):
    """EnvManager.reset_idx for the robot-only scene (env_manager.py:273-301).  ``mask`` bool [N].
    Mutates st; afterwards the derived states of ALL envs are refreshed
    (base_multirotor.py:204-205) iff any env was reset."""
    if not bool(mask.any()):
        return
    dt_ = st.root.dtype
    T = lambda x: torch.tensor(x, dtype=dt_)
    m1 = mask.unsqueeze(1)
    # IGE_env_manager.py:513-519
    st.bounds_min = torch.where(m1, _lerp_rand(T(model.bounds_lower_range[0]), T(model.bounds_lower_range[1]), draws.bounds_lo), st.bounds_min)
    st.bounds_max = torch.where(m1, _lerp_rand(T(model.bounds_upper_range[0]), T(model.bounds_upper_range[1]), draws.bounds_hi), st.bounds_max)
    # base_multirotor.py:177-199
    rs = _lerp_rand(T(model.min_init_state), T(model.max_init_state), draws.state)
    pos = st.bounds_min + (st.bounds_max - st.bounds_min) * rs[:, 0:3]  # torch_interpolate_ratio
    quat = quat_from_euler_xyz(rs[:, 3], rs[:, 4], rs[:, 5])
    new_root = torch.cat([pos, quat, rs[:, 7:10], rs[:, 10:13]], dim=1)
    st.root = torch.where(m1, new_root, st.root)
    if model.randomize_params:  # base_lee_controller.py:101-118
        st.K_pos = torch.where(m1, _lerp_rand(T(model.K_pos_range[0]), T(model.K_pos_range[1]), draws.K_pos), st.K_pos)
        st.K_vel = torch.where(m1, _lerp_rand(T(model.K_vel_range[0]), T(model.K_vel_range[1]), draws.K_vel), st.K_vel)
        st.K_rot = torch.where(m1, _lerp_rand(T(model.K_rot_range[0]), T(model.K_rot_range[1]), draws.K_rot), st.K_rot)
        st.K_angvel = torch.where(m1, _lerp_rand(T(model.K_angvel_range[0]), T(model.K_angvel_range[1]), draws.K_angvel), st.K_angvel)
    # motor_model.py:140-154
    st.tau_inc = torch.where(m1, _lerp_rand(T(model.tau_inc_range[0]), T(model.tau_inc_range[1]), draws.tau_inc), st.tau_inc)
    st.tau_dec = torch.where(m1, _lerp_rand(T(model.tau_dec_range[0]), T(model.tau_dec_range[1]), draws.tau_dec), st.tau_dec)
    st.thrust = torch.where(m1, _lerp_rand(T(float(model.min_thrust)), T(float(model.max_thrust)), draws.thrust), st.thrust)
    if model.use_rps:
        st.k_thrust = torch.where(m1, _lerp_rand(T(model.k_thrust_range[0]), T(model.k_thrust_range[1]), draws.k_thrust), st.k_thrust)
    st.sim_steps = torch.where(mask, torch.zeros_like(st.sim_steps), st.sim_steps)
    st.derived = update_states(st.root)


# --------------------------------------------------------------------------------------
# whole env step of the position task
# --------------------------------------------------------------------------------------
def position_task_step(
    model: Hp1Model,
    st: Hp1State,
    actions,
    target,
    episode_len_steps: int = 500,
    physics_steps: int = 1,
    draws: Optional[ResetDraws] = None,
    draw_fn=None,
):
    """PositionSetpointTask.step (:152-182) over EnvManager.step (env_manager.py:399-432).

    Resets use ``draws`` if given, else ``draw_fn()`` is called ONLY when some env resets
    (RNG consumption pattern of the reference).  Returns (obs, reward, terminations,
    truncations, reset_mask)."""
    N = actions.shape[0]
    crashes = torch.zeros(N, dtype=torch.bool)
    for _ in range(physics_steps):
        physics_step(model, st, actions)
        # compute_observations(): contact-force collision flag -- robot-only scene has no contacts
    st.sim_steps = st.sim_steps + 1
    reward, crashes = position_task_reward(st, target, crashes)
    trunc = st.sim_steps > episode_len_steps
    reset_mask = crashes | trunc
    if bool(reset_mask.any()):
        if draws is None:
            draws = draw_fn()
        reset_envs(model, st, reset_mask, draws)
    obs = position_task_obs(st, target)
    return obs, reward, crashes, trunc, reset_mask
