"""Oracle of the contact between free obstacles (agx_obstacle_obstacle_contact; DESIGN.md "Contact mode", "Contact between free
obstacles").  TEST INFRASTRUCTURE ONLY.  contact_core.cuh's obstacle_box_world, obstacle_box_near, obstacle_box_pair,
obstacle_contacts_solve and contact_body_store restated in numpy float32 scalars, every operation in the header's order, so that
it matches the kernel bit for bit:

* ``box_world``: an asset row's box in the world (centre, axes, half extents, bounding radius).
* ``box_pair``: the separating-axis test, the axis choice and the contact manifold of one pair -> (contacts, axis kind).
* ``env_contact``: one env as obstacle_obstacle_contact_kernel runs it: bodies, pairs (i, j) in order until the list is full, the
  sequential-impulse solve and the write-back.
* ``box_signed_distance``: float64 signed distance of points to a box, for the brute-force checks."""
import numpy as np

f32 = np.float32
CONTACT_MAX = 8
MAX_CONTACTS = 128  # AGX_OBSTACLE_MAX_CONTACTS
AXIS_TOL = f32(1e-4)
ZERO, ONE, HALF, TWO = f32(0.0), f32(1.0), f32(0.5), f32(2.0)


def _dot(a, b):
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]


def _cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def _matvec(M, x):
    return [M[3 * i] * x[0] + M[3 * i + 1] * x[1] + M[3 * i + 2] * x[2] for i in range(3)]


def _quat_R(q):
    x, y, z, w = q
    return [ONE - TWO * (y * y + z * z), TWO * (x * y - z * w), TWO * (x * z + y * w),
            TWO * (x * y + z * w), ONE - TWO * (x * x + z * z), TWO * (y * z - x * w),
            TWO * (x * z - y * w), TWO * (y * z + x * w), ONE - TWO * (x * x + y * y)]


def _fminmax(x, lo, hi):
    return min(max(x, lo), hi)


class Body:
    """contact_body_load of an asset row and its AgxObstacleMass row [13]"""

    def __init__(self, row, m):
        row, m = [f32(v) for v in row[:13]], [f32(v) for v in m]
        self.x, self.q, self.v, self.w = row[0:3], row[3:7], row[7:10], row[10:13]
        R = _quat_R(self.q)
        cm = _matvec(R, m[1:4])
        self.c = [self.x[k] + cm[k] for k in range(3)]
        self.oc = [self.x[k] - self.c[k] for k in range(3)]
        ii = m[4:13]
        A = [R[3 * i] * ii[j] + R[3 * i + 1] * ii[3 + j] + R[3 * i + 2] * ii[6 + j] for i in range(3) for j in range(3)]
        self.Iw = [A[3 * i] * R[3 * j] + A[3 * i + 1] * R[3 * j + 1] + A[3 * i + 2] * R[3 * j + 2] for i in range(3) for j in range(3)]
        self.inv_m = m[0]
        self.free = bool(m[0] > 0) or any(v != 0 for v in ii)

    def apply(self, P, s):  # cbody_apply
        dw = _matvec(self.Iw, _cross(s, P))
        dwx = _cross(dw, self.oc)
        self.w = [self.w[k] + dw[k] for k in range(3)]
        self.v = [self.v[k] + (P[k] * self.inv_m + dwx[k]) for k in range(3)]


def _keff(r, d, inv_m, Iw):
    rd = _cross(r, d)
    return inv_m + _dot(rd, _matvec(Iw, rd))


def _vel(v, w, r):
    wr = _cross(w, r)
    return [v[k] + wr[k] for k in range(3)]


def box_world(row, box):
    """obstacle_box_world: row [>=13], box [15] -> dict(c, a (three axes), h, r)"""
    row, box = [f32(v) for v in row[:7]], [f32(v) for v in box]
    R = _quat_R(row[3:7])
    t = _matvec(R, box[0:3])
    b = {"c": [row[k] + t[k] for k in range(3)], "a": [_matvec(R, box[3 + 3 * k:6 + 3 * k]) for k in range(3)], "h": box[12:15]}
    b["r"] = np.sqrt(_dot(b["h"], b["h"]))
    return b


def box_near(P, A, B):
    d = [B["c"][k] - A["c"][k] for k in range(3)]
    s = A["r"] + B["r"] + f32(P.contact_offset)
    return bool(_dot(d, d) <= s * s)


def _sep(A, B, d, L):
    rA, rB = ZERO, ZERO
    for k in range(3):
        rA = rA + A["h"][k] * abs(_dot(A["a"][k], L))
        rB = rB + B["h"][k] * abs(_dot(B["a"][k], L))
    return abs(_dot(d, L)) - (rA + rB)


def box_pair(P, A, B):
    """obstacle_box_pair -> (contacts [(p, n, depth)], kind): kind 'none', 'faceA', 'faceB' or 'edge'"""
    d = [B["c"][k] - A["c"][k] for k in range(3)]
    co = f32(P.contact_offset)
    sA = sB = sE = ZERO
    kA = kB = 0
    kE = -1
    for k in range(3):
        s = _sep(A, B, d, A["a"][k])
        if s > co:
            return [], "none"
        if k == 0 or s > sA:
            sA, kA = s, k
    for k in range(3):
        s = _sep(A, B, d, B["a"][k])
        if s > co:
            return [], "none"
        if k == 0 or s > sB:
            sB, kB = s, k
    LE = [ZERO] * 3
    for i in range(3):
        for j in range(3):
            L = _cross(A["a"][i], B["a"][j])
            l2 = _dot(L, L)
            if l2 < f32(1e-6):
                continue
            inv = ONE / np.sqrt(l2)
            L = [L[k] * inv for k in range(3)]
            s = _sep(A, B, d, L)
            if s > co:
                return [], "none"
            if kE < 0 or s > sE:
                sE, kE, LE = s, 3 * i + j, L
    refB = bool(sB > sA + AXIS_TOL)
    sF = sB if refB else sA
    if kE >= 0 and sE > sF + AXIS_TOL:
        i, j = kE // 3, kE % 3
        sg = ONE if _dot(d, LE) >= ZERO else -ONE
        n = [LE[k] * sg for k in range(3)]
        pa, pb = list(A["c"]), list(B["c"])
        for m in range(3):
            if m != i:
                s = A["h"][m] if _dot(A["a"][m], n) >= ZERO else -A["h"][m]
                pa = [pa[k] + A["a"][m][k] * s for k in range(3)]
            if m != j:
                s = -B["h"][m] if _dot(B["a"][m], n) > ZERO else B["h"][m]
                pb = [pb[k] + B["a"][m][k] * s for k in range(3)]
        da, db = A["a"][i], B["a"][j]
        w = [pa[k] - pb[k] for k in range(3)]
        b, dd, e = _dot(da, db), _dot(da, w), _dot(db, w)
        den = ONE - b * b
        ta = _fminmax((b * e - dd) / den, -A["h"][i], A["h"][i])
        tb = _fminmax((e - b * dd) / den, -B["h"][j], B["h"][j])
        p = [((pa[k] + da[k] * ta) + (pb[k] + db[k] * tb)) * HALF for k in range(3)]
        return [(p, n, -sE)], "edge"
    R, I = (B, A) if refB else (A, B)
    kr = kB if refB else kA
    sg = ONE if _dot(d, R["a"][kr]) >= ZERO else -ONE
    n = [R["a"][kr][k] * sg for k in range(3)]
    nr = [-n[k] for k in range(3)] if refB else list(n)
    fc = [R["c"][k] + nr[k] * R["h"][kr] for k in range(3)]
    r1, r2 = (kr + 1) % 3, (kr + 2) % 3
    t1, t2, e1, e2 = R["a"][r1], R["a"][r2], R["h"][r1], R["h"][r2]
    m, best = 0, abs(_dot(nr, I["a"][0]))
    for k in (1, 2):
        v = abs(_dot(nr, I["a"][k]))
        if v > best:
            best, m = v, k
    so = -I["h"][m] if _dot(nr, I["a"][m]) > ZERO else I["h"][m]
    u, v = (m + 1) % 3, (m + 2) % 3
    poly = []
    for su, sv in ((ONE, ONE), (-ONE, ONE), (-ONE, -ONE), (ONE, -ONE)):
        rel = [((I["c"][k] + I["a"][m][k] * so) + I["a"][u][k] * (su * I["h"][u]) + I["a"][v][k] * (sv * I["h"][v])) - fc[k]
               for k in range(3)]
        poly.append([_dot(rel, t1), _dot(rel, t2), _dot(rel, nr)])
    for pl in range(4):
        if not poly:
            break
        ax = pl >> 1
        sgn, lim = (-ONE if pl & 1 else ONE), (e2 if ax else e1)
        out = []
        for q in range(len(poly)):
            pc, pp = poly[q], poly[q - 1]
            dc, dp = pc[ax] * sgn - lim, pp[ax] * sgn - lim
            if (dc <= ZERO) != (dp <= ZERO):
                t = dp / (dp - dc)
                out.append([pp[k] + (pc[k] - pp[k]) * t for k in range(3)])
            if dc <= ZERO:
                out.append(list(pc))
        poly = out
    cands = []
    for q, pq in enumerate(poly):
        if pq[2] > co:
            continue
        hs = pq[2] * HALF
        p = [fc[k] + t1[k] * pq[0] + t2[k] * pq[1] + nr[k] * hs for k in range(3)]
        cands.append((pq[2], q, (p, n, -pq[2])))
    cands.sort(key=lambda c: (c[0], c[1]))  # contact_insert: key s, ties to the lower index
    return [c[2] for c in cands[:CONTACT_MAX]], ("faceB" if refB else "faceA")


def solve(P, bodies, L):
    """obstacle_contacts_solve on bodies (Body, changed in place) and the list L [(p, n, depth, i, j)]"""
    rest, dt, maxd, mu = f32(P.rest_offset), f32(P.dt), f32(P.max_depenetration_velocity), f32(P.friction)
    st = []
    for p, n, depth, i, j in L:
        bi, bj = bodies[i], bodies[j]
        si = [p[k] - bi.c[k] for k in range(3)]
        sj = [p[k] - bj.c[k] for k in range(3)]
        kn = _keff(sj, n, bj.inv_m, bj.Iw) + _keff(si, n, bi.inv_m, bi.Iw)
        bias = min(max(depth - rest, ZERO) / dt, maxd)
        st.append({"kn": kn, "bias": bias, "ln": ZERO, "lt": [ZERO] * 3})
    for _ in range(int(P.iterations)):
        for (p, nn, depth, i, j), o in zip(L, st):
            bi, bj = bodies[i], bodies[j]
            ri = [p[k] - bi.x[k] for k in range(3)]
            rj = [p[k] - bj.x[k] for k in range(3)]
            si = [p[k] - bi.c[k] for k in range(3)]
            sj = [p[k] - bj.c[k] for k in range(3)]
            vr, u = _vel(bj.v, bj.w, rj), _vel(bi.v, bi.w, ri)
            vr = [vr[k] - u[k] for k in range(3)]
            dl = (o["bias"] - _dot(nn, vr)) / o["kn"]
            l1 = max(o["ln"] + dl, ZERO)
            dl = l1 - o["ln"]
            o["ln"] = l1
            dP = [nn[k] * dl for k in range(3)]
            nP = [-x for x in dP]
            if bj.free:
                bj.apply(dP, sj)
            if bi.free:
                bi.apply(nP, si)
            vr, u = _vel(bj.v, bj.w, rj), _vel(bi.v, bi.w, ri)
            vr = [vr[k] - u[k] for k in range(3)]
            vn = _dot(nn, vr)
            vt = [vr[k] - nn[k] * vn for k in range(3)]
            l2 = list(o["lt"])
            s = np.sqrt(_dot(vt, vt))
            if s > ZERO:
                t = [vt[k] / s for k in range(3)]
                dt_ = s / (_keff(sj, t, bj.inv_m, bj.Iw) + _keff(si, t, bi.inv_m, bi.Iw))
                l2 = [l2[k] - t[k] * dt_ for k in range(3)]
            mag, lim = np.sqrt(_dot(l2, l2)), mu * o["ln"]
            if mag > lim:
                f = lim / mag
                l2 = [l2[k] * f for k in range(3)]
            dP = [l2[k] - o["lt"][k] for k in range(3)]
            o["lt"] = l2
            nP = [-x for x in dP]
            if bj.free:
                bj.apply(dP, sj)
            if bi.free:
                bi.apply(nP, si)


def store(b, row, dt):
    """contact_body_store: the body's new twist and the first-order pose correction, into row (float32 array, in place)"""
    dt = f32(dt)
    old_v, old_w = [f32(x) for x in row[7:10]], [f32(x) for x in row[10:13]]
    h = [(b.w[k] - old_w[k]) * dt * HALF for k in range(3)]
    q = b.q
    qn = [q[0] + h[0] * q[3] + h[1] * q[2] - h[2] * q[1], q[1] - h[0] * q[2] + h[1] * q[3] + h[2] * q[0],
          q[2] + h[0] * q[1] - h[1] * q[0] + h[2] * q[3], q[3] - h[0] * q[0] - h[1] * q[1] - h[2] * q[2]]
    inv = ONE / np.sqrt(qn[0] * qn[0] + qn[1] * qn[1] + qn[2] * qn[2] + qn[3] * qn[3])
    for k in range(3):
        row[k] = b.x[k] + (b.v[k] - old_v[k]) * dt
    for k in range(4):
        row[3 + k] = qn[k] * inv
    row[7:10], row[10:13] = b.v, b.w


def env_contact(P, rows, mass, boxes, asset_box, max_contacts=MAX_CONTACTS):
    """one env of agx_obstacle_obstacle_contact: rows [A,>=13] (copied), mass [A,13], boxes [F,15], asset_box [A] ->
    (rows, list [(p, n, depth, i, j)], kinds {(i, j): kind} of the pairs that reached the narrow phase)"""
    rows = np.array(rows, dtype=f32, copy=True)
    A = rows.shape[0]
    bodies = [Body(rows[a], mass[a]) for a in range(A)]
    X = [box_world(rows[a], boxes[asset_box[a]]) for a in range(A)]
    L, kinds, full = [], {}, False
    for i in range(A):
        for j in range(i + 1, A):
            if not (bodies[i].free or bodies[j].free) or not box_near(P, X[i], X[j]):
                continue
            c, kinds[(i, j)] = box_pair(P, X[i], X[j])
            if not c:
                continue
            if len(L) + len(c) > max_contacts:
                full = True
                break
            L += [(p, n, dep, i, j) for p, n, dep in c]
        if full:
            break
    if L:
        solve(P, bodies, L)
        touched = {i for *_, i, _ in L} | {j for *_, j in L}
        for a in sorted(touched):
            if bodies[a].free:
                store(bodies[a], rows[a], P.dt)
    return rows, L, kinds


def box_signed_distance(points, c, axes, h):
    """float64 signed distance of points [n,3] to the box (centre c, axes [3,3] as rows, half extents h): < 0 inside"""
    local = (np.asarray(points, np.float64) - np.asarray(c, np.float64)) @ np.asarray(axes, np.float64).T
    q = np.abs(local) - np.asarray(h, np.float64)
    return np.linalg.norm(np.maximum(q, 0.0), axis=1) + np.minimum(q.max(axis=1), 0.0)
