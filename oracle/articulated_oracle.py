"""Float64 checker of the articulated-multirotor dynamics (DESIGN.md "Articulated robots").

An independent restatement: the joint-space equations of motion are ASSEMBLED -- the mass matrix by the composite-rigid-body sum
M = sum_i J_i^T I_i J_i over the bodies' Jacobians, the bias C by the recursive Newton-Euler pass with zero accelerations -- and the
implicit-drive system (M + diag(0_6, dt d + dt^2 k)) [a0; qdd] = tau_explicit - C is solved with numpy.linalg.solve.  Nothing here
follows the articulated-body recursion of articulated_core.cuh.

Conventions shared with the product (they define what is compared, not how it is computed): spatial vectors in world axes about the
base origin O, angular part first; generalised velocity = (base twist at O, q-dot); a0 = the base's spatial acceleration at O.
`table` is a dict of numpy arrays with the fields of AgxArticulation (num_bodies, parent, joint_R [B,3,3], joint_p, axis, mass, com,
inertia [B,3,3], stiffness, damping, motor_body, motor_R [M,3,3], motor_p, motor_torque; integrate() also reads lower, upper,
limited [B]).

substep() is one whole sub-step of the articulated step (articulated_core.cuh's art_env_step): the controller, allocation, motor
model, drag and derived states of oracle/hp1_oracle.py run in float64, then dynamics() and integrate() below."""
import numpy as np
import torch

from . import hp1_oracle as HO


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


def _quat_mul(a, b):
    """Hamilton product of xyzw quaternions"""
    av, aw, bv, bw = a[:3], a[3], b[:3], b[3]
    return np.concatenate([aw * bv + bw * av + np.cross(av, bv), [aw * bw - av @ bv]])


def integrate(model, table, root, a0, q, qd, qdd):
    """DESIGN.md section 3 on the base with the ABA's accelerations, then the joints of section 6 "Integration", one env.
    model: hp1_oracle.Hp1Model (dt, damping, caps).  -> (root' [13], q' [D], qd' [D], q_free [D] = q' before the limit projection)"""
    dt = model.dt
    root = np.asarray(root, np.float64)
    x, quat, v, w = root[0:3], root[3:7], root[7:10], root[10:13]
    R = quat_to_matrix(quat)
    a = a0[3:] + np.cross(w, v)  # the classical acceleration of the base origin
    v1 = (v + dt * a) * max(0.0, 1.0 - dt * model.linear_damping)
    vn = np.linalg.norm(v1)
    if vn > model.max_linear_velocity:
        v1 = v1 * (model.max_linear_velocity / vn)
    W = R.T @ w
    W1 = W + dt * (R.T @ a0[:3])
    w1 = (R @ W1) * max(0.0, 1.0 - dt * model.angular_damping)
    wn = np.linalg.norm(w1)
    if wn > model.max_angular_velocity:
        w1 = w1 * (model.max_angular_velocity / wn)
        wn = np.linalg.norm(w1)
    x1 = x + dt * v1
    so = np.sin(0.5 * dt * wn) / wn if wn > 0 else 0.0
    qn = _quat_mul(np.concatenate([w1 * so, [np.cos(0.5 * dt * wn)]]), quat)
    qn = qn / np.linalg.norm(qn)
    # joints: semi-implicit, then the projection onto [lower, upper] of a limited joint
    v1j = qd + dt * qdd
    q1 = q + dt * v1j
    q_free = q1.copy()
    B = int(table["num_bodies"])
    for j in range(B - 1):
        if table["limited"][j + 1]:
            lo, hi = table["lower"][j + 1], table["upper"][j + 1]
            if q1[j] <= lo:
                q1[j], v1j[j] = lo, max(v1j[j], 0.0)
            if q1[j] >= hi:
                q1[j], v1j[j] = hi, min(v1j[j], 0.0)
    return np.concatenate([x1, qn, v1, w1]), q1, v1j, q_free


def substep(model, table, st, q, qd, qs, qds, actions, disturbance=None):
    """One sub-step of the articulated step for N envs in float64.

    model: hp1_oracle.Hp1Model of the engine's MultirotorSpec; st: hp1_oracle.Hp1State in float64 (root [N,13], thrust and the
    motor constants / gains the kernel reads); q, qd, qs, qds [N,D]; actions [N,A]; disturbance: [N,6] body-frame wrench or None.
    The drag and disturbance act at the base origin, rotated to world axes.
    -> dict: root [N,13], q, qd, q_free [N,D], thrust [N,M], derived (update_states at the sub-step's start), a0 [N,6], qdd [N,D]"""
    f64 = lambda a: torch.as_tensor(np.asarray(a), dtype=torch.float64)
    root = st.root
    N, D = root.shape[0], int(table["num_bodies"]) - 1
    d = HO.update_states(root)
    cmd = HO.controller_wrench(model, st, d, torch.clamp(f64(actions), -10.0, 10.0))
    ref = cmd if model.controller == HO.CTRL_NONE else cmd @ model.pinv_allocation(torch.float64).T
    thrust = HO.motor_update(model, st, ref)
    df, dtq = HO.drag_wrench(model, d)
    if disturbance is not None:
        df, dtq = df + f64(disturbance)[:, 0:3], dtq + f64(disturbance)[:, 3:6]
    F_w, T_w = HO.quat_rotate(root[:, 3:7], df).numpy(), HO.quat_rotate(root[:, 3:7], dtq).numpy()
    q, qd, qs, qds = (np.asarray(a, np.float64).reshape(N, D) for a in (q, qd, qs, qds))
    out = {k: np.zeros(s) for k, s in (("root", (N, 13)), ("q", (N, D)), ("qd", (N, D)), ("q_free", (N, D)), ("a0", (N, 6)),
                                        ("qdd", (N, D)))}
    r, th = root.numpy(), thrust.numpy()
    for n in range(N):
        a0, qdd = dynamics(table, r[n], q[n], qd[n], qs[n], qds[n], model.dt, model.gravity, th[n], F_w[n], T_w[n])
        out["a0"][n], out["qdd"][n] = a0, qdd
        out["root"][n], out["q"][n], out["qd"][n], out["q_free"][n] = integrate(model, table, r[n], a0, q[n], qd[n], qdd)
    out["thrust"], out["derived"] = th, {k: v.numpy() for k, v in d.items()}
    return out


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
