"""Float64 checker of the articulated-multirotor dynamics with torque-driven (effort-mode) joints (DESIGN.md "Articulated robots",
"Torque-driven joints"), on top of oracle/articulated_oracle.py.  `table` is the same dict of numpy arrays with the fields of
AgxArticulation; an effort DOF's entries there have stiffness 0 and damping = the URDF <dynamics damping> alone.

The joint-space system is assembled exactly as articulated_oracle.dynamics assembles it (CRBA mass matrix, RNEA bias), and the
commanded torque enters its right-hand side:
    (M + diag(0_6, dt d + dt^2 k)) [a0; qdd] = tau - C,
    tau_j = k_j (qs_j - q_j - dt qd_j) + d_j (qds_j - qd_j)   for a position DOF,
    tau_j = clamp(e_j, -E_j, E_j) - d_j qd_j                  for an effort DOF (unclamped where E_j = 0).
Nothing here follows the articulated-body recursion of articulated_core.cuh."""
import numpy as np

from . import articulated_imu_oracle as IO
from . import hp1_oracle as HO
from .articulated_oracle import _crf, _crm, body_inertia, integrate, kinematics


def effort_torque(e, limit):
    """tau_e = e clamped to +-limit where limit > 0, e where limit = 0"""
    e, limit = np.asarray(e, np.float64), np.asarray(limit, np.float64)
    return np.where(limit > 0, np.clip(e, -limit, limit), e)


def system(table, root, q, qd, dt, grav, thrust, F_w, T_w):
    """(H [6+D, 6+D], C [6+D]): the implicit-drive matrix M + diag(0_6, dt d + dt^2 k) and the bias of articulated_oracle.dynamics"""
    B = int(table["num_bodies"])
    D = B - 1
    n = 6 + D
    root = np.asarray(root, np.float64)
    R, P, S = kinematics(table, root[3:7], q)
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
    return H, C


def joint_torque(table, q, qd, qs, qds, dt, effort_dof, effort, effort_limit):
    """[D] the explicit joint torque: the drive of a position DOF, tau_e - d qd of an effort DOF"""
    B = int(table["num_bodies"])
    k, d = np.asarray(table["stiffness"][1:B], np.float64), np.asarray(table["damping"][1:B], np.float64)
    drive = k * (qs - q - dt * qd) + d * (qds - qd)
    return np.where(np.asarray(effort_dof, bool), effort_torque(effort, effort_limit) - d * qd, drive)


def dynamics(table, root, q, qd, qs, qds, dt, grav, thrust, F_w, T_w, effort_dof, effort, effort_limit):
    """-> (a0 [6], qdd [D]): articulated_oracle.dynamics' inputs plus the effort DOFs (bool [D]), their commands and limits [D]"""
    q, qd, qs, qds = (np.asarray(a, np.float64) for a in (q, qd, qs, qds))
    H, C = system(table, root, q, qd, dt, grav, thrust, F_w, T_w)
    tau = np.zeros(H.shape[0])
    tau[6:] = joint_torque(table, q, qd, qs, qds, dt, effort_dof, effort, effort_limit)
    x = np.linalg.solve(H, tau - C)
    return x[:6], x[6:]


def substep(model, table, st, q, qd, qs, qds, actions, effort_dof, effort, effort_limit, disturbance=None):
    """articulated_oracle.substep with effort DOFs: effort [N,D] the commands, effort_dof / effort_limit [D].  -> the same dict"""
    thrust, F_w, T_w = IO.substep_inputs(model, st, actions, disturbance)
    root = st.root
    d = HO.update_states(root)
    N, D = root.shape[0], int(table["num_bodies"]) - 1
    q, qd, qs, qds, effort = (np.asarray(a, np.float64).reshape(N, D) for a in (q, qd, qs, qds, effort))
    out = {k: np.zeros(s) for k, s in (("root", (N, 13)), ("q", (N, D)), ("qd", (N, D)), ("q_free", (N, D)), ("a0", (N, 6)),
                                        ("qdd", (N, D)))}
    r = root.numpy()
    for n in range(N):
        a0, qdd = dynamics(table, r[n], q[n], qd[n], qs[n], qds[n], model.dt, model.gravity, thrust[n], F_w[n], T_w[n], effort_dof,
                           effort[n], effort_limit)
        out["a0"][n], out["qdd"][n] = a0, qdd
        out["root"][n], out["q"][n], out["qd"][n], out["q_free"][n] = integrate(model, table, r[n], a0, q[n], qd[n], qdd)
    out["thrust"], out["derived"] = thrust, {k: v.numpy() for k, v in d.items()}
    return out
