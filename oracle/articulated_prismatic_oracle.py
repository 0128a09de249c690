"""Float64 checker of articulated multirotors with prismatic joints (DESIGN.md "Articulated robots", "Prismatic joints"), beside
oracle/articulated_oracle.py and its siblings.  `table` is the same dict of numpy arrays with the fields of AgxArticulation, plus
"prismatic" [B] bool: body i's joint is prismatic, a translation of body i by q along a = R_parent joint_R_i axis_i (R_i =
R_parent joint_R_i, P_i = P_parent + R_parent joint_p_i + a q, motion subspace S_i = (0, a)).  Without that column every joint is
revolute, and every function here gives its sibling's result bit for bit: each restates its sibling's assembly with the
kinematics below.

The same independent method as the siblings: the mass matrix by the composite-rigid-body sum over the bodies' Jacobians, the bias by
the recursive Newton-Euler pass with zero accelerations, the implicit-drive system solved with numpy.linalg.solve (with the effort
DOFs of articulated_effort_oracle), the joint forces by the Newton-Euler backward recursion of articulated_joint_force_oracle.  The
bias term V_i x (S_i qd_i) holds for a slider too: its a is fixed in the parent, so dS_i/dt = V_parent x S_i = V_i x S_i.
Nothing here follows the articulated-body recursion of articulated_core.cuh."""
import numpy as np

from . import articulated_effort_oracle as EO
from . import articulated_imu_oracle as IO
from . import articulated_joint_force_oracle as JO
from . import hp1_oracle as HO
from .articulated_body_state_oracle import matrix_to_quat
from .articulated_oracle import _crf, _crm, _rot, body_inertia, integrate, quat_to_matrix


def _slides(table, i):
    p = table.get("prismatic")
    return p is not None and bool(p[i])


def kinematics(table, quat, q):
    """(R [B,3,3], P [B,3] relative to the base origin, S [B,6] world joint motion subspaces, row 0 unused)"""
    B = int(table["num_bodies"])
    R, P, S = np.zeros((B, 3, 3)), np.zeros((B, 3)), np.zeros((B, 6))
    R[0] = quat_to_matrix(quat)
    for i in range(1, B):
        l = int(table["parent"][i])
        RJ = R[l] @ table["joint_R"][i]
        if _slides(table, i):
            a = RJ @ table["axis"][i]
            R[i], P[i] = RJ, P[l] + R[l] @ table["joint_p"][i] + a * q[i - 1]
            S[i, 3:] = a
            continue
        R[i] = RJ @ _rot(table["axis"][i], q[i - 1])
        P[i] = P[l] + R[l] @ table["joint_p"][i]
        a = RJ @ table["axis"][i]
        S[i, :3], S[i, 3:] = a, np.cross(P[i], a)
    return R, P, S


def system(table, root, q, qd, dt, grav, thrust, F_w, T_w):
    """(H [6+D, 6+D], C [6+D]): the implicit-drive matrix M + diag(0_6, dt d + dt^2 k) and the bias (articulated_effort_oracle.system)"""
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


def dynamics(table, root, q, qd, qs, qds, dt, grav, thrust, F_w, T_w, effort_dof=None, effort=None, effort_limit=None):
    """-> (a0 [6], qdd [D]) of one sub-step (articulated_effort_oracle.dynamics; effort_dof None: no effort DOF).  A prismatic
    DOF's drive and effort are forces: the same laws, in N"""
    q, qd, qs, qds = (np.asarray(a, np.float64) for a in (q, qd, qs, qds))
    D = int(table["num_bodies"]) - 1
    if effort_dof is None:
        effort_dof, effort, effort_limit = np.zeros(D, bool), np.zeros(D), np.zeros(D)
    H, C = system(table, root, q, qd, dt, grav, thrust, F_w, T_w)
    tau = np.zeros(H.shape[0])
    tau[6:] = EO.joint_torque(table, q, qd, qs, qds, dt, effort_dof, effort, effort_limit)
    x = np.linalg.solve(H, tau - C)
    return x[:6], x[6:]


def body_motion(table, root, q, qd, a0, qdd):
    """(R, P, V [B,6], A [B,6]) of every body, world axes about O (articulated_imu_oracle.body_motion)"""
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


def newton_euler(table, root, q, qd, a0, qdd, grav, thrust, F_w, T_w):
    """-> (f [B,6] the parent's wrench on each body, world axes about O, f[0] = the base's residual; R; P)
    (articulated_joint_force_oracle.newton_euler)"""
    B = int(table["num_bodies"])
    R, P, V, A = body_motion(table, root, q, qd, a0, qdd)
    fext = JO.external_forces(table, R, P, grav, thrust, F_w, T_w)
    f = np.zeros((B, 6))
    for i in range(B):
        I = body_inertia(float(table["mass"][i]), P[i] + R[i] @ table["com"][i], R[i] @ table["inertia"][i] @ R[i].T)
        f[i] = I @ A[i] + _crf(V[i]) @ (I @ V[i]) - fext[i]
    for i in range(B - 1, 0, -1):
        f[int(table["parent"][i])] += f[i]
    return f, R, P


def rows(table, f, R, P):
    """-> (wrench [B,6] in each body's frame, force then torque about the joint origin, row 0 zero; dof [D]): a revolute DOF's
    force is axis . (the torque), a prismatic DOF's axis . (the force)"""
    W, _ = JO.rows(table, f, R, P)
    B = int(table["num_bodies"])
    return W, np.array([float(table["axis"][i] @ (W[i, :3] if _slides(table, i) else W[i, 3:])) for i in range(1, B)])


def joint_force(table, root, q, qd, qs, qds, dt, grav, thrust, F_w, T_w, effort_dof=None, effort=None, effort_limit=None):
    """-> dict: wrench [B,6], dof [D], a0 [6], qdd [D], residual [6] (articulated_joint_force_oracle.joint_force)"""
    q, qd = np.asarray(q, np.float64), np.asarray(qd, np.float64)
    a0, qdd = dynamics(table, root, q, qd, qs, qds, dt, grav, thrust, F_w, T_w, effort_dof, effort, effort_limit)
    f, R, P = newton_euler(table, root, q, qd, a0, qdd, grav, thrust, F_w, T_w)
    W, dof = rows(table, f, R, P)
    return {"wrench": W, "dof": dof, "a0": a0, "qdd": qdd, "residual": f[0].copy()}


def body_states(table, root, q, qd):
    """-> [B,13] per-body rows of one env, laid out like a root_state row (articulated_body_state_oracle.body_states)"""
    B = int(table["num_bodies"])
    root = np.asarray(root, np.float64)
    q, qd = np.asarray(q, np.float64), np.asarray(qd, np.float64)
    R, P, S = kinematics(table, root[3:7], q)
    V = np.zeros((B, 6))
    V[0] = np.concatenate([root[10:13], root[7:10]])
    out = np.zeros((B, 13))
    out[0] = root[:13]
    for i in range(1, B):
        V[i] = V[int(table["parent"][i])] + S[i] * qd[i - 1]
        out[i, 0:3] = root[0:3] + P[i]
        out[i, 3:7] = matrix_to_quat(R[i])
        out[i, 7:10] = V[i, 3:] + np.cross(V[i, :3], P[i])
        out[i, 10:13] = V[i, :3]
    return out


def momentum(table, root, q, qd):
    """(linear momentum, angular momentum about the system COM), world frame (articulated_oracle.momentum)"""
    B = int(table["num_bodies"])
    root = np.asarray(root, np.float64)
    R, P, S = kinematics(table, root[3:7], q)
    v = np.concatenate([root[10:13], root[7:10]])
    vs, h, mt, cs = [None] * B, np.zeros(6), 0.0, np.zeros(3)
    for i in range(B):
        vs[i] = v if i == 0 else vs[int(table["parent"][i])] + S[i] * qd[i - 1]
        m = float(table["mass"][i])
        c = P[i] + R[i] @ table["com"][i]
        h += body_inertia(m, c, R[i] @ table["inertia"][i] @ R[i].T) @ vs[i]
        mt += m
        cs += m * c
    com = cs / mt
    return h[3:], h[:3] - np.cross(com, h[3:])


def substep(model, table, st, q, qd, qs, qds, actions, effort_dof=None, effort=None, effort_limit=None, disturbance=None):
    """one whole sub-step for N envs in float64 (articulated_effort_oracle.substep): -> dict root [N,13], q, qd, q_free [N,D],
    thrust [N,M], derived, a0 [N,6], qdd [N,D].  integrate() is articulated_oracle's: a limited slider is projected as a revolute
    joint is"""
    thrust, F_w, T_w = IO.substep_inputs(model, st, actions, disturbance)
    root = st.root
    d = HO.update_states(root)
    N, D = root.shape[0], int(table["num_bodies"]) - 1
    q, qd, qs, qds = (np.asarray(a, np.float64).reshape(N, D) for a in (q, qd, qs, qds))
    effort = np.zeros((N, D)) if effort is None else np.asarray(effort, np.float64).reshape(N, D)
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
