"""Float64 checker of the joint forces of an articulated multirotor (DESIGN.md "Articulated robots", "Joint force sensing"), on top of
oracle/articulated_oracle.py and oracle/articulated_effort_oracle.py.  `table` is the same dict of numpy arrays with the fields of
AgxArticulation.

The generalised accelerations come from the assembled CRBA + RNEA solve (articulated_effort_oracle.dynamics, which is
articulated_oracle.dynamics where no DOF is in effort mode); each body's spatial velocity V_i and acceleration A_i follow from them
(articulated_imu_oracle.body_motion).  The joint forces are then an independent Newton-Euler backward recursion -- no articulated
inertia of the kernel's ABA: in world axes about the base origin O, angular first, the wrench body i's parent exerts on it is
    f_i = I_i A_i + V_i x* I_i V_i  -  f_ext,i  +  sum over the children c of i of f_c,
its rate of momentum, minus gravity, the motors on it (and on the base the drag and disturbance), plus what it passes on to its
children.  For the floating base the same sum is the residual of its Newton-Euler balance, zero to rounding.  Body i's row is
    (R_i^T F, R_i^T (n_O - P_i x F))  for f_i = (n_O; F),
and its DOF force axis_i . (that torque)."""
import numpy as np

from . import articulated_effort_oracle as EO
from . import articulated_imu_oracle as IO
from .articulated_oracle import _crf, body_inertia


def external_forces(table, R, P, grav, thrust, F_w, T_w):
    """[B,6]: gravity at each COM, every motor's thrust and reaction torque on its body, the drag + disturbance on the base"""
    B = int(table["num_bodies"])
    fext = np.zeros((B, 6))
    for i in range(B):
        c = P[i] + R[i] @ table["com"][i]
        fg = float(table["mass"][i]) * np.asarray(grav, np.float64)
        fext[i] += np.concatenate([np.cross(c, fg), fg])
    for k in range(len(thrust)):
        b = int(table["motor_body"][k])
        ez = (R[b] @ table["motor_R"][k])[:, 2]
        pos = P[b] + R[b] @ table["motor_p"][k]
        f = ez * thrust[k]
        fext[b] += np.concatenate([np.cross(pos, f) + ez * table["motor_torque"][k] * thrust[k], f])
    fext[0] += np.concatenate([np.asarray(T_w, np.float64), np.asarray(F_w, np.float64)])
    return fext


def newton_euler(table, root, q, qd, a0, qdd, grav, thrust, F_w, T_w):
    """-> (f [B,6] world axes about O, the parent's wrench on each body; f[0] = the base's residual; R, P): the backward recursion"""
    B = int(table["num_bodies"])
    R, P, V, A = IO.body_motion(table, root, q, qd, a0, qdd)
    fext = external_forces(table, R, P, grav, thrust, F_w, T_w)
    f = np.zeros((B, 6))
    for i in range(B):
        I = body_inertia(float(table["mass"][i]), P[i] + R[i] @ table["com"][i], R[i] @ table["inertia"][i] @ R[i].T)
        f[i] = I @ A[i] + _crf(V[i]) @ (I @ V[i]) - fext[i]
    for i in range(B - 1, 0, -1):  # children have larger indices than their parents
        f[int(table["parent"][i])] += f[i]
    return f, R, P


def rows(table, f, R, P):
    """-> (wrench [B,6] in each body's frame, row 0 zero; dof [D])"""
    B = int(table["num_bodies"])
    W = np.zeros((B, 6))
    for i in range(1, B):
        n, F = f[i, :3], f[i, 3:]
        W[i, :3], W[i, 3:] = R[i].T @ F, R[i].T @ (n - np.cross(P[i], F))
    return W, np.array([float(table["axis"][i] @ W[i, 3:]) for i in range(1, B)])


def joint_force(table, root, q, qd, qs, qds, dt, grav, thrust, F_w, T_w, effort_dof=None, effort=None, effort_limit=None):
    """-> dict: wrench [B,6], dof [D], a0 [6], qdd [D], residual [6] (the base's Newton-Euler balance, world axes about O) of one
    sub-step at (root, q, qd); effort_dof / effort / effort_limit as articulated_effort_oracle.dynamics (None: no effort DOF)"""
    D = int(table["num_bodies"]) - 1
    q, qd = np.asarray(q, np.float64), np.asarray(qd, np.float64)
    if effort_dof is None:
        effort_dof, effort, effort_limit = np.zeros(D, bool), np.zeros(D), np.zeros(D)
    a0, qdd = EO.dynamics(table, root, q, qd, qs, qds, dt, grav, thrust, F_w, T_w, effort_dof, effort, effort_limit)
    f, R, P = newton_euler(table, root, q, qd, a0, qdd, grav, thrust, F_w, T_w)
    W, dof = rows(table, f, R, P)
    return {"wrench": W, "dof": dof, "a0": a0, "qdd": qdd, "residual": f[0].copy()}


def drive_torque(table, q, qd, qs, qds, qdd, dt, effort_dof=None, effort=None, effort_limit=None):
    """[D] the identity dof_force satisfies: k (qs - q') + d (qds - qd') of a position DOF, tau_e - d qd' of an effort DOF, at the
    unprojected end-of-step state qd' = qd + dt qdd, q' = q + dt qd'"""
    B = int(table["num_bodies"])
    k, d = np.asarray(table["stiffness"][1:B], np.float64), np.asarray(table["damping"][1:B], np.float64)
    v1 = np.asarray(qd, np.float64) + dt * np.asarray(qdd, np.float64)
    q1 = np.asarray(q, np.float64) + dt * v1
    pos = k * (np.asarray(qs, np.float64) - q1) + d * (np.asarray(qds, np.float64) - v1)
    if effort_dof is None:
        return pos
    return np.where(np.asarray(effort_dof, bool), EO.effort_torque(effort, effort_limit) - d * v1, pos)


def substep(model, table, st, q, qd, qs, qds, actions, disturbance=None, effort_dof=None, effort=None, effort_limit=None):
    """the joint forces of N envs for the sub-step starting at (st.root, q, qd): dict with wrench [N,B,6], dof [N,D], a0 [N,6],
    qdd [N,D], residual [N,6], thrust [N,M]; effort [N,D] the commands where effort_dof is given"""
    thrust, F_w, T_w = IO.substep_inputs(model, st, actions, disturbance)
    r = st.root.numpy()
    N, B = r.shape[0], int(table["num_bodies"])
    D = B - 1
    q, qd, qs, qds = (np.asarray(a, np.float64).reshape(N, D) for a in (q, qd, qs, qds))
    eff = np.zeros((N, D)) if effort is None else np.asarray(effort, np.float64).reshape(N, D)
    out = {"wrench": np.zeros((N, B, 6)), "dof": np.zeros((N, D)), "a0": np.zeros((N, 6)), "qdd": np.zeros((N, D)),
           "residual": np.zeros((N, 6)), "thrust": thrust}
    for n in range(N):
        o = joint_force(table, r[n], q[n], qd[n], qs[n], qds[n], model.dt, model.gravity, thrust[n], F_w[n], T_w[n], effort_dof,
                        eff[n], effort_limit)
        for k in ("wrench", "dof", "a0", "qdd", "residual"):
            out[k][n] = o[k]
    return out
