"""Oracle of the obstacle-ground contact (agx_obstacle_ground_contact; DESIGN.md "Contact mode", "Ground contact of free obstacles").
TEST INFRASTRUCTURE ONLY.  contact_core.cuh's obstacle_ground_row restated in numpy float32, vectorised over rows, every operation
in the header's order, so that it matches the kernel bit for bit:

* ``select``: the reach test, the kinematic test, the world vertices and the kept contacts (the AGX_CONTACT_MAX deepest vertices
  below contact_offset, ties to the lower vertex index).
* ``solve``: the one-body sequential-impulse solve against the ground at rest and the write-back (contact_body_load,
  cbody_apply, contact_body_store, as oracle/contact_dynamic_oracle.py restates them).
* ``ground_contact``: both, on rows [R,>=13] with their mass entries and file indices.
* ``lowest_vertex``: the lowest world vertex height of each row (float64), for the checks."""
import numpy as np

from .contact_dynamic_oracle import _keff, _quat_R, _vel, _world_inv_inertia
from .contact_oracle import CONTACT_MAX, _cross, _dot, _matvec, _where

f32 = np.float32


def _world(rows, verts):
    """world positions of verts [V,3] (asset frame) for every row [r,13]: (x + R v) per component, [r,V] each, float32"""
    R = [c[:, None] for c in _quat_R([rows[:, 3 + k] for k in range(4)])]
    rv = _matvec(R, [verts[None, :, k] for k in range(3)])
    return [rows[:, k, None] + rv[k] for k in range(3)]


def select(P, rows, mass, vertices, file_offset, file_reach, asset_file):
    """rows [R,>=13], mass [R,13], hull tables (vertices [V,3], file_offset [F+1], file_reach [F]), asset_file [R] ->
    kept [R,CONTACT_MAX] vertex indices deepest first (-1 unused), count [R], contacts [R,CONTACT_MAX,7] (p, n, depth)"""
    rows, mass = np.asarray(rows, f32), np.asarray(mass, f32)
    vertices, off = np.asarray(vertices, f32).reshape(-1, 3), np.asarray(file_offset)
    reach, af = np.asarray(file_reach, f32), np.asarray(asset_file).reshape(-1)
    Rn = rows.shape[0]
    kept = np.full((Rn, CONTACT_MAX), -1, np.int64)
    count = np.zeros(Rn, np.int64)
    cts = np.zeros((Rn, CONTACT_MAX, 7), f32)
    co = f32(P.contact_offset)
    near = ~(rows[:, 2] - reach[af] > co)
    free = (mass[:, 0] > 0) | (mass[:, 4:13] != 0).any(axis=1)
    for f in np.unique(af):
        sel = np.nonzero((af == f) & near & free)[0]
        v = vertices[off[f]:off[f + 1]]
        if len(sel) == 0 or len(v) == 0:
            continue
        p = _world(rows[sel], v)
        z = p[2]
        cand = z < co
        idx = np.broadcast_to(np.arange(len(v)), z.shape)
        order = np.lexsort((idx, np.where(cand, z, np.inf)), axis=-1)[:, :CONTACT_MAX]  # (key z, vertex index) ascending
        n = np.minimum(cand.sum(axis=1), CONTACT_MAX)
        for j in range(order.shape[1]):
            m = j < n
            r, o = sel[m], order[m, j]
            kept[r, j] = o
            pr = np.nonzero(m)[0]
            for k in range(3):
                cts[r, j, k] = p[k][pr, o]
            cts[r, j, 5] = 1.0
            cts[r, j, 6] = -z[pr, o]
        count[sel] = n
    return kept, count, cts


def solve(P, rows, mass, contacts, count):
    """rows [R,>=13] (copied), mass [R,13], contacts [R,CONTACT_MAX,7], count [R] -> rows with every row with count > 0 solved and
    written back (the rows select() kept contacts for are free)"""
    rows = np.array(rows, dtype=f32, copy=True)
    mass, contacts, count = np.asarray(mass, f32), np.asarray(contacts, f32), np.asarray(count)
    rest, dt, maxd, mu = f32(P.rest_offset), f32(P.dt), f32(P.max_depenetration_velocity), f32(P.friction)
    zero, half = f32(0.0), f32(0.5)
    x, q = [rows[:, k] for k in range(3)], [rows[:, 3 + k] for k in range(4)]
    v, w = [rows[:, 7 + k] for k in range(3)], [rows[:, 10 + k] for k in range(3)]
    R = _quat_R(q)
    cm = _matvec(R, [mass[:, 1 + k] for k in range(3)])
    c = [x[k] + cm[k] for k in range(3)]
    oc = [x[k] - c[k] for k in range(3)]
    inv_m = mass[:, 0]
    Iw = _world_inv_inertia(R, [mass[:, 4 + k] for k in range(9)])
    S = range(CONTACT_MAX)
    act = [count > i for i in S]
    nrm = [[contacts[:, i, 3 + k] for k in range(3)] for i in S]
    ra = [[contacts[:, i, k] - x[k] for k in range(3)] for i in S]
    sa = [[contacts[:, i, k] - c[k] for k in range(3)] for i in S]
    zeros = np.zeros(rows.shape[0], f32)

    def apply(m, Pv, s, v, w):  # cbody_apply where m
        dw = _matvec(Iw, _cross(s, Pv))
        dwx = _cross(dw, oc)
        return _where(m, [v[k] + (Pv[k] * inv_m + dwx[k]) for k in range(3)], v), _where(m, [w[k] + dw[k] for k in range(3)], w)

    with np.errstate(all="ignore"):
        kn = [_keff(sa[i], nrm[i], inv_m, Iw) for i in S]
        bias = [np.minimum(np.maximum(contacts[:, i, 6] - rest, zero) / dt, maxd) for i in S]
        ln = [zeros.copy() for _ in S]
        lt = [[zeros.copy() for _ in range(3)] for _ in S]
        for _ in range(int(P.iterations)):
            for i in S:
                m, nn = act[i], nrm[i]
                vr = _vel(v, w, ra[i])
                dl = (bias[i] - _dot(nn, vr)) / kn[i]
                l1 = np.maximum(ln[i] + dl, zero)
                dl = l1 - ln[i]
                ln[i] = np.where(m, l1, ln[i])
                v, w = apply(m, [nn[k] * dl for k in range(3)], sa[i], v, w)
                vr = _vel(v, w, ra[i])
                vn = _dot(nn, vr)
                vt = [vr[k] - nn[k] * vn for k in range(3)]
                s = np.sqrt(_dot(vt, vt))
                t = [vt[k] / s for k in range(3)]
                dt_ = s / _keff(sa[i], t, inv_m, Iw)
                l2 = _where(s > zero, [lt[i][k] - t[k] * dt_ for k in range(3)], lt[i])
                mag, lim = np.sqrt(_dot(l2, l2)), mu * ln[i]
                f = lim / mag
                l2 = _where(mag > lim, [l2[k] * f for k in range(3)], l2)
                dP = [l2[k] - lt[i][k] for k in range(3)]
                lt[i] = _where(m, l2, lt[i])
                v, w = apply(m, dP, sa[i], v, w)
        # contact_body_store
        wr = count > 0
        h = [(w[k] - rows[:, 10 + k]) * dt * half for k in range(3)]
        qn = [q[0] + h[0] * q[3] + h[1] * q[2] - h[2] * q[1],
              q[1] - h[0] * q[2] + h[1] * q[3] + h[2] * q[0],
              q[2] + h[0] * q[1] - h[1] * q[0] + h[2] * q[3],
              q[3] - h[0] * q[0] - h[1] * q[1] - h[2] * q[2]]
        inv = f32(1.0) / np.sqrt(qn[0] * qn[0] + qn[1] * qn[1] + qn[2] * qn[2] + qn[3] * qn[3])
        new = rows.copy()
        for k in range(3):
            new[:, k] = x[k] + (v[k] - rows[:, 7 + k]) * dt
            new[:, 7 + k] = v[k]
            new[:, 10 + k] = w[k]
        for k in range(4):
            new[:, 3 + k] = qn[k] * inv
    rows[wr] = new[wr]
    return rows


def ground_contact(P, rows, mass, vertices, file_offset, file_reach, asset_file):
    """one launch of agx_obstacle_ground_contact on rows [R,>=13] -> (rows, kept, count); inputs are not modified"""
    kept, count, cts = select(P, rows, mass, vertices, file_offset, file_reach, asset_file)
    return solve(P, rows, mass, cts, count), kept, count


def lowest_vertex(rows, vertices, file_offset, asset_file):
    """lowest world vertex height of each row [R], float64"""
    rows, af = np.asarray(rows, np.float64), np.asarray(asset_file).reshape(-1)
    out = np.full(rows.shape[0], np.inf)
    for f in np.unique(af):
        sel = np.nonzero(af == f)[0]
        v = np.asarray(vertices, np.float64).reshape(-1, 3)[file_offset[f]:file_offset[f + 1]]
        if len(v):
            out[sel] = np.stack(_world(rows[sel], v))[2].min(axis=1)
    return out
