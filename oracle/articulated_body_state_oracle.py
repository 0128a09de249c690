"""Float64 checker of the per-body state of an articulated multirotor (DESIGN.md "Articulated robots", "Body states"), on top of
oracle/articulated_oracle.py's kinematics().  `table` is the same dict of numpy arrays with the fields of AgxArticulation."""
import numpy as np

from .articulated_oracle import kinematics


def matrix_to_quat(R):
    """xyzw quaternion of a rotation matrix (Shepperd's method); its sign is not normalised"""
    t = np.trace(R)
    if t > 0:
        s = 2.0 * np.sqrt(1.0 + t)
        return np.array([(R[2, 1] - R[1, 2]) / s, (R[0, 2] - R[2, 0]) / s, (R[1, 0] - R[0, 1]) / s, 0.25 * s])
    i = int(np.argmax(np.diag(R)))
    j, k = (i + 1) % 3, (i + 2) % 3
    s = 2.0 * np.sqrt(1.0 + R[i, i] - R[j, j] - R[k, k])
    v = np.zeros(4)
    v[i], v[j], v[k], v[3] = 0.25 * s, (R[j, i] + R[i, j]) / s, (R[k, i] + R[i, k]) / s, (R[k, j] - R[j, k]) / s
    return v


def body_states(table, root, q, qd):
    """-> [B,13] per-body rows of one env, laid out like a root_state row: world position of the body-frame origin, xyzw quaternion
    body -> world, world linear velocity of the origin, world angular velocity.  Row 0 is `root`.  Velocities: the spatial velocity at
    the base origin V_i = V_parent + S_i q-dot_i (V_0 = (w, v) of the root row); the origin of body i moves with V_lin + w_i x P_i."""
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
