"""Float64 checker of the articulated-multirotor dynamics (DESIGN.md "Articulated robots").

An independent restatement: the joint-space equations of motion are ASSEMBLED -- the mass matrix by the composite-rigid-body sum
M = sum_i J_i^T I_i J_i over the bodies' Jacobians, the bias C by the recursive Newton-Euler pass with zero accelerations -- and the
implicit-drive system (M + diag(0_6, dt d + dt^2 k)) [a0; qdd] = tau_explicit - C is solved with numpy.linalg.solve.  Nothing here
follows the articulated-body recursion of articulated_core.cuh.

Conventions shared with the product (they define what is compared, not how it is computed): spatial vectors in world axes about the
base origin O, angular part first; generalised velocity = (base twist at O, q-dot); a0 = the base's spatial acceleration at O.
`table` is a dict of numpy arrays with the fields of AgxArticulation (num_bodies, parent, joint_R [B,3,3], joint_p, axis, mass, com,
inertia [B,3,3], stiffness, damping, motor_body, motor_R [M,3,3], motor_p, motor_torque)."""
import numpy as np


def _skew(v):
    return np.array([[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]])


def _rot(axis, t):
    a = np.asarray(axis, np.float64)
    K = _skew(a)
    return np.eye(3) + np.sin(t) * K + (1.0 - np.cos(t)) * (K @ K)


def quat_to_matrix(q):
    x, y, z, w = (float(v) for v in q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def _crm(v):
    w, u = _skew(v[:3]), _skew(v[3:])
    X = np.zeros((6, 6))
    X[:3, :3], X[3:, :3], X[3:, 3:] = w, u, w
    return X


def _crf(v):
    return -_crm(v).T


def kinematics(table, quat, q):
    """(R [B,3,3], P [B,3] relative to the base origin, S [B,6] world joint motion subspaces, row 0 unused)"""
    B = int(table["num_bodies"])
    R, P, S = np.zeros((B, 3, 3)), np.zeros((B, 3)), np.zeros((B, 6))
    R[0] = quat_to_matrix(quat)
    for i in range(1, B):
        l = int(table["parent"][i])
        RJ = R[l] @ table["joint_R"][i]
        R[i] = RJ @ _rot(table["axis"][i], q[i - 1])
        P[i] = P[l] + R[l] @ table["joint_p"][i]
        a = RJ @ table["axis"][i]
        S[i, :3], S[i, 3:] = a, np.cross(P[i], a)
    return R, P, S


def body_inertia(m, c, Ic):
    I = np.zeros((6, 6))
    C = _skew(c)
    I[:3, :3] = Ic + m * (C @ C.T)
    I[:3, 3:], I[3:, :3], I[3:, 3:] = m * C, m * C.T, m * np.eye(3)
    return I


def dynamics(table, root, q, qd, qs, qds, dt, grav, thrust, F_w, T_w):
    """-> (a0 [6], qdd [D]) of one sub-step: the same inputs as articulated_core.cuh's art_dynamics"""
    B = int(table["num_bodies"])
    D = B - 1
    n = 6 + D
    root = np.asarray(root, np.float64)
    R, P, S = kinematics(table, root[3:7], q)
    # Jacobians: body i moves with the base and every joint on its path to the root
    J = np.zeros((B, 6, n))
    for i in range(B):
        J[i, :, :6] = np.eye(6)
        k = i
        while k > 0:
            J[i, :, 6 + k - 1] = S[k]
            k = int(table["parent"][k])
    nu = np.concatenate([root[10:13], root[7:10], qd])
    I = np.zeros((B, 6, 6))
    fext = np.zeros((B, 6))
    for i in range(B):
        m = float(table["mass"][i])
        c = P[i] + R[i] @ table["com"][i]
        I[i] = body_inertia(m, c, R[i] @ table["inertia"][i] @ R[i].T)
        fg = m * np.asarray(grav, np.float64)
        fext[i] += np.concatenate([np.cross(c, fg), fg])
    for k in range(len(thrust)):
        b = int(table["motor_body"][k])
        Rm = R[b] @ table["motor_R"][k]
        ez = Rm[:, 2]
        pos = P[b] + R[b] @ table["motor_p"][k]
        f = ez * thrust[k]
        fext[b] += np.concatenate([np.cross(pos, f) + ez * table["motor_torque"][k] * thrust[k], f])
    fext[0] += np.concatenate([T_w, F_w])
    # RNEA with zero accelerations: a_i = a_parent + v_i x (S_i qd_i)
    v, a, C = np.zeros((B, 6)), np.zeros((B, 6)), np.zeros(n)
    for i in range(B):
        v[i] = J[i] @ nu
        if i > 0:
            l = int(table["parent"][i])
            a[i] = a[l] + _crm(v[i]) @ (S[i] * qd[i - 1])
        f = I[i] @ a[i] + _crf(v[i]) @ (I[i] @ v[i]) - fext[i]
        C += J[i].T @ f
    M = sum(J[i].T @ I[i] @ J[i] for i in range(B))
    k, d = np.asarray(table["stiffness"][1:B], np.float64), np.asarray(table["damping"][1:B], np.float64)
    H = M.copy()
    H[6:, 6:] += np.diag(dt * d + dt * dt * k)
    tau = np.zeros(n)
    tau[6:] = k * (qs - q - dt * qd) + d * (qds - qd)
    x = np.linalg.solve(H, tau - C)
    return x[:6], x[6:]


def momentum(table, root, q, qd):
    """(linear momentum, angular momentum about the system COM), world frame"""
    B = int(table["num_bodies"])
    root = np.asarray(root, np.float64)
    R, P, S = kinematics(table, root[3:7], q)
    v = np.concatenate([root[10:13], root[7:10]])
    vs, h, mt, cs = [None] * B, np.zeros(6), 0.0, np.zeros(3)
    for i in range(B):
        if i == 0:
            vs[i] = v
        else:
            vs[i] = vs[int(table["parent"][i])] + S[i] * qd[i - 1]
        m = float(table["mass"][i])
        c = P[i] + R[i] @ table["com"][i]
        h += body_inertia(m, c, R[i] @ table["inertia"][i] @ R[i].T) @ vs[i]
        mt += m
        cs += m * c
    com = cs / mt
    L = h[:3] - np.cross(com, h[3:])  # angular momentum about O -> about the COM
    return h[3:], L
