"""Float64 checker of the IMU input of one body of an articulated multirotor (DESIGN.md "Articulated robots", "IMU on a link"), on top
of oracle/articulated_oracle.py's kinematics() and dynamics().  `table` is the same dict of numpy arrays with the fields of
AgxArticulation.

The generalised accelerations come from dynamics() (the assembled CRBA + RNEA system, not the articulated-body recursion of the
kernel); each body's spatial acceleration is then A_i = A_parent + S_i qdd_i + V_i x (S_i qd_i), V_i = V_parent + S_i qd_i (world axes
about the base origin O, angular first).  From them, for body b with rotation R, origin P (relative to O), mass m, COM com and
inertia I (about the COM, body axes):
    c = P + R com,   a_c = A_lin + alpha x c + w x (V_lin + w x c)      (the classical acceleration of the COM)
    f = m R^T (a_c - g),   n = I R^T alpha + w_b x I w_b,   w_b = R^T w."""
import numpy as np
import torch

from . import hp1_oracle as HO
from .articulated_oracle import _crm, dynamics, kinematics


def body_motion(table, root, q, qd, a0, qdd):
    """(R [B,3,3], P [B,3], V [B,6], A [B,6]): every body's rotation, origin relative to O, spatial velocity and spatial
    acceleration, world axes about O"""
    B = int(table["num_bodies"])
    root = np.asarray(root, np.float64)
    R, P, S = kinematics(table, root[3:7], q)
    V, A = np.zeros((B, 6)), np.zeros((B, 6))
    V[0], A[0] = np.concatenate([root[10:13], root[7:10]]), np.asarray(a0, np.float64)
    for i in range(1, B):
        l = int(table["parent"][i])
        vj = S[i] * qd[i - 1]
        V[i] = V[l] + vj
        A[i] = A[l] + S[i] * qdd[i - 1] + _crm(V[i]) @ vj
    return R, P, V, A


def com_acceleration(table, i, R, P, V, A):
    """(c, a_c): body i's COM relative to O and its classical acceleration"""
    c = P[i] + R[i] @ table["com"][i]
    w = V[i, :3]
    return c, A[i, 3:] + np.cross(A[i, :3], c) + np.cross(w, V[i, 3:] + np.cross(w, c))


def body_forces(table, root, q, qd, a0, qdd, grav):
    """[B,3]: m_i (a_c,i - g) of every body, world axes -- the non-gravitational force on each body, joint reactions included"""
    B = int(table["num_bodies"])
    R, P, V, A = body_motion(table, root, q, qd, a0, qdd)
    g = np.asarray(grav, np.float64)
    return np.array([float(table["mass"][i]) * (com_acceleration(table, i, R, P, V, A)[1] - g) for i in range(B)])


def imu_from_motion(table, b, grav, R, P, V, A):
    """[9] = (f, n, w_b) of body b, its frame"""
    _, ac = com_acceleration(table, b, R, P, V, A)
    Rb, I = R[b], np.asarray(table["inertia"][b], np.float64)
    wb, ab = Rb.T @ V[b, :3], Rb.T @ A[b, :3]
    f = float(table["mass"][b]) * (Rb.T @ (ac - np.asarray(grav, np.float64)))
    n = I @ ab + np.cross(wb, I @ wb)
    return np.concatenate([f, n, wb])


def imu_input(table, root, q, qd, qs, qds, dt, grav, thrust, F_w, T_w, b):
    """-> [9] (f_b, n_b, w_b) of body b at the state (root, q, qd): the same inputs as dynamics() plus the body"""
    q, qd = np.asarray(q, np.float64), np.asarray(qd, np.float64)
    a0, qdd = dynamics(table, root, q, qd, qs, qds, dt, grav, thrust, F_w, T_w)
    return imu_from_motion(table, b, grav, *body_motion(table, root, q, qd, a0, qdd))


def substep_inputs(model, st, actions, disturbance=None):
    """the controller -> allocation -> motor model -> drag of one sub-step (articulated_oracle.substep's), float64:
    -> (thrust [N,M], F_w [N,3], T_w [N,3]) -- the motor thrusts and the base's drag + disturbance force / torque in world axes"""
    f64 = lambda a: torch.as_tensor(np.asarray(a), dtype=torch.float64)
    root = st.root
    d = HO.update_states(root)
    cmd = HO.controller_wrench(model, st, d, torch.clamp(f64(actions), -10.0, 10.0))
    ref = cmd if model.controller == HO.CTRL_NONE else cmd @ model.pinv_allocation(torch.float64).T
    thrust = HO.motor_update(model, st, ref)
    df, dtq = HO.drag_wrench(model, d)
    if disturbance is not None:
        df, dtq = df + f64(disturbance)[:, 0:3], dtq + f64(disturbance)[:, 3:6]
    return thrust.numpy(), HO.quat_rotate(root[:, 3:7], df).numpy(), HO.quat_rotate(root[:, 3:7], dtq).numpy()


def substep_imu(model, table, st, q, qd, qs, qds, actions, b, disturbance=None):
    """the IMU input of body b for N envs, the sub-step starting at (st.root, q, qd): [N,9], and the dict of per-env extras
    (thrust [N,M], F_w [N,3], a0 [N,6], qdd [N,D])"""
    thrust, F_w, T_w = substep_inputs(model, st, actions, disturbance)
    r = st.root.numpy()
    N, D = r.shape[0], int(table["num_bodies"]) - 1
    q, qd, qs, qds = (np.asarray(a, np.float64).reshape(N, D) for a in (q, qd, qs, qds))
    out, a0s, qdds = np.zeros((N, 9)), np.zeros((N, 6)), np.zeros((N, D))
    for n in range(N):
        a0, qdd = dynamics(table, r[n], q[n], qd[n], qs[n], qds[n], model.dt, model.gravity, thrust[n], F_w[n], T_w[n])
        a0s[n], qdds[n] = a0, qdd
        out[n] = imu_from_motion(table, b, model.gravity, *body_motion(table, r[n], q[n], qd[n], a0, qdd))
    return out, {"thrust": thrust, "F_w": F_w, "T_w": T_w, "a0": a0s, "qdd": qdds}
