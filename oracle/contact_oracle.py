"""Oracle of the rigid contact mode (agx_hp2_contact; DESIGN.md "Contact mode").  TEST INFRASTRUCTURE ONLY.

* ``find_contacts``: brute force -- for every object the closest point over all of its world triangles (float64), the ground plane,
  the AGX_CONTACT_MAX nearest by (distance, object index), the ground last on ties.
* ``solve``: contact_core.cuh's sequential-impulse solve restated in numpy float32, vectorised over envs, every operation in the
  header's order (no FMA anywhere), so it matches the kernel's arithmetic bit for bit given the same contact list.
* ``simulate``: a free sphere under gravity, stepped like an env sub-step (semi-implicit Euler as the robot integrator, then the
  contact search and the solve), for the physical checks.

``P`` is anything with the fields of AgxContactParams (radius, contact_offset, rest_offset, dt, mass, inertia_inv[9], com[3],
friction, max_depenetration_velocity, force_threshold, iterations, ground_plane)."""
import numpy as np

CONTACT_MAX = 8
f32 = np.float32


def _dot(a, b):
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]


def _cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def _matvec(M, x):
    return [M[3 * i] * x[0] + M[3 * i + 1] * x[1] + M[3 * i + 2] * x[2] for i in range(3)]


def _where(m, new, old):
    return [np.where(m, a, b) for a, b in zip(new, old)]


def solve(P, root, contacts, count):
    """root [E,>=13] float32 (copied), contacts [E,CONTACT_MAX,7] (point, normal, depth), count [E] -> (root, force [E,3], crash [E])"""
    root = np.array(root, dtype=f32, copy=True)
    contacts = np.asarray(contacts, f32)
    count = np.asarray(count)
    E = root.shape[0]
    ii, com_b = [f32(v) for v in P.inertia_inv], [f32(v) for v in P.com]
    rest, dt, maxd, mu = f32(P.rest_offset), f32(P.dt), f32(P.max_depenetration_velocity), f32(P.friction)
    x, y, z, qw = (root[:, 3 + k] for k in range(4))
    one, two, zero = f32(1.0), f32(2.0), f32(0.0)
    R = [one - two * (y * y + z * z), two * (x * y - z * qw), two * (x * z + y * qw),
         two * (x * y + z * qw), one - two * (x * x + z * z), two * (y * z - x * qw),
         two * (x * z - y * qw), two * (y * z + x * qw), one - two * (x * x + y * y)]
    com = _matvec(R, com_b)
    com = [root[:, k] + com[k] for k in range(3)]
    A = [R[3 * i] * ii[j] + R[3 * i + 1] * ii[3 + j] + R[3 * i + 2] * ii[6 + j] for i in range(3) for j in range(3)]
    Iw = [A[3 * i] * R[3 * j] + A[3 * i + 1] * R[3 * j + 1] + A[3 * i + 2] * R[3 * j + 2] for i in range(3) for j in range(3)]
    inv_m = one / f32(P.mass)
    v = [root[:, 7 + k] for k in range(3)]
    w = [root[:, 10 + k] for k in range(3)]

    def keff(r, d):
        rd = _cross(r, d)
        return inv_m + _dot(rd, _matvec(Iw, rd))

    def apply(m, Pv, r, v, w):
        dw = _matvec(Iw, _cross(r, Pv))
        return _where(m, [v[k] + Pv[k] * inv_m for k in range(3)], v), _where(m, [w[k] + dw[k] for k in range(3)], w)

    def vel(v, w, r):
        wr = _cross(w, r)
        return [v[k] + wr[k] for k in range(3)]

    S = range(CONTACT_MAX)
    act = [count > i for i in S]
    nrm = [[contacts[:, i, 3 + k] for k in range(3)] for i in S]
    r = [[contacts[:, i, k] - com[k] for k in range(3)] for i in S]
    zeros = np.zeros(E, f32)
    with np.errstate(all="ignore"):
        kn = [keff(r[i], nrm[i]) for i in S]
        bias = [np.minimum(np.maximum(contacts[:, i, 6] - rest, zero) / dt, maxd) for i in S]
        ln = [zeros.copy() for _ in S]
        lt = [[zeros.copy() for _ in range(3)] for _ in S]
        for _ in range(int(P.iterations)):
            for i in S:
                m, nn = act[i], nrm[i]
                vr = vel(v, w, r[i])
                dl = (bias[i] - _dot(nn, vr)) / kn[i]
                l1 = np.maximum(ln[i] + dl, zero)
                dl = l1 - ln[i]
                ln[i] = np.where(m, l1, ln[i])
                v, w = apply(m, [nn[k] * dl for k in range(3)], r[i], v, w)
                vr = vel(v, w, r[i])
                vn = _dot(nn, vr)
                vt = [vr[k] - nn[k] * vn for k in range(3)]
                s = np.sqrt(_dot(vt, vt))
                t = [vt[k] / s for k in range(3)]
                dt_ = s / keff(r[i], t)
                l2 = _where(s > zero, [lt[i][k] - t[k] * dt_ for k in range(3)], lt[i])
                mag, lim = np.sqrt(_dot(l2, l2)), mu * ln[i]
                f = lim / mag
                l2 = _where(mag > lim, [l2[k] * f for k in range(3)], l2)
                dP = [l2[k] - lt[i][k] for k in range(3)]
                lt[i] = _where(m, l2, lt[i])
                v, w = apply(m, dP, r[i], v, w)
    imp = [zeros.copy() for _ in range(3)]
    for i in S:
        imp = _where(act[i], [imp[k] + nrm[i][k] * ln[i] + lt[i][k] for k in range(3)], imp)
    force = np.stack([imp[k] / dt for k in range(3)], axis=1)
    crash = (count > 0) & (np.sqrt(_dot([force[:, 0], force[:, 1], force[:, 2]], [force[:, 0], force[:, 1], force[:, 2]])) > f32(P.force_threshold))
    force[count == 0] = 0.0
    for k in range(3):
        root[:, 7 + k] = v[k]
        root[:, 10 + k] = w[k]
    return root, force, crash


def closest_points(p, tris):
    """closest point on each triangle (rows a, ab, ac) to p, float64, Ericson's Voronoi regions -> (q [n,3], d2 [n])"""
    t = np.asarray(tris, np.float64).reshape(-1, 3, 3)
    a, ab, ac = t[:, 0], t[:, 1], t[:, 2]
    p = np.asarray(p, np.float64)
    b, c = a + ab, a + ac
    d1, d2 = (ab * (p - a)).sum(1), (ac * (p - a)).sum(1)
    d3, d4 = (ab * (p - b)).sum(1), (ac * (p - b)).sum(1)
    d5, d6 = (ab * (p - c)).sum(1), (ac * (p - c)).sum(1)
    vc, vb, va = d1 * d4 - d3 * d2, d5 * d2 - d1 * d6, d3 * d6 - d5 * d4
    with np.errstate(all="ignore"):
        q_ab = a + ab * (d1 / (d1 - d3))[:, None]
        q_ac = a + ac * (d2 / (d2 - d6))[:, None]
        q_bc = b + (c - b) * ((d4 - d3) / ((d4 - d3) + (d5 - d6)))[:, None]
        den = 1.0 / (va + vb + vc)
        q_in = a + ab * (vb * den)[:, None] + ac * (vc * den)[:, None]
    masks = [(d1 <= 0) & (d2 <= 0), (d3 >= 0) & (d4 <= d3), (vc <= 0) & (d1 >= 0) & (d3 <= 0), (d6 >= 0) & (d5 <= d6),
             (vb <= 0) & (d2 >= 0) & (d6 <= 0), (va <= 0) & ((d4 - d3) >= 0) & ((d5 - d6) >= 0)]
    q = np.select([m[:, None] for m in masks], [a, b, q_ab, c, q_ac, q_bc], q_in)
    return q, ((p - q) ** 2).sum(1)


def find_contacts(P, centres, objects, return_ambiguous=False):
    """centres [E,3]; objects[e] = list of [n,9] world triangle arrays (a, ab, ac), one per object in index order.
    -> contacts [E,CONTACT_MAX,7] float32, count [E], ids [E,CONTACT_MAX] (object index, len(objects[e]) = ground, -1 unused)
    return_ambiguous: also [E] bool -- a kept contact is ill-conditioned in float32: its object has a second closest point
    elsewhere within 20 µm + 1e-4 relative of the closest distance (a centre near a medial plane of a solid: which one rounding picks
    is arbitrary), or the centre is within 1 mm of the surface (the normal (c - q) / |c - q| loses most of its bits)."""
    E = len(centres)
    out = np.zeros((E, CONTACT_MAX, 7), f32)
    count = np.zeros(E, np.int32)
    ids = np.full((E, CONTACT_MAX), -1, np.int32)
    ambiguous = np.zeros(E, bool)
    reach = f32(P.radius) + f32(P.contact_offset)
    for e in range(E):
        c = np.asarray(centres[e], f32)
        cands = []
        for k, tris in enumerate(objects[e]):
            if len(tris) == 0:
                continue
            q, d2 = closest_points(c, tris)
            j = int(np.argmin(d2))
            if not d2[j] <= float(reach) ** 2:
                continue
            dist = np.sqrt(d2[j])
            if dist > 0:
                nv = (c - q[j]) / dist
            else:
                t = np.asarray(tris[j], np.float64).reshape(3, 3)
                nv = np.cross(t[1], t[2])
                nv /= np.linalg.norm(nv)
            near = (np.sqrt(d2) <= dist * (1 + 1e-4) + 2e-5) & (np.abs(q - q[j]).max(axis=1) > 1e-4)
            cands.append((dist, k, np.concatenate([q[j], nv, [float(P.radius) - dist]]), bool(near.any()) or dist < 1e-3))
        if P.ground_plane and c[2] <= reach:
            cands.append((float(c[2]), len(objects[e]), np.array([c[0], c[1], 0.0, 0.0, 0.0, 1.0, float(P.radius) - float(c[2])]), False))
        cands.sort(key=lambda t: (t[0], t[1]))
        cands = cands[:CONTACT_MAX]
        count[e] = len(cands)
        for i, (_, k, row, amb) in enumerate(cands):
            out[e, i], ids[e, i] = row, k
            ambiguous[e] |= amb
    return (out, count, ids, ambiguous) if return_ambiguous else (out, count, ids)


def simulate(P, x, v, w, steps, gravity=(0.0, 0.0, -9.81), objects=()):
    """one sphere (centre of mass at its centre), `steps` sub-steps of: v += g dt, x += v dt (the robot integrator's order, no
    damping), contact search against `objects` (world triangle arrays) and the ground, solve.  The orientation stays the identity:
    with the centre of mass at the centre and an isotropic inertia nothing in the contact depends on it.
    Returns per sub-step: x, v after the integration (before the solve), v and w after the solve, the contact force."""
    root = np.zeros((1, 13), f32)
    root[0, 0:3], root[0, 6], root[0, 7:10], root[0, 10:13] = x, 1.0, v, w
    g, dt = np.asarray(gravity, f32), f32(P.dt)
    hist = {k: [] for k in ("x", "v_pre", "v", "w", "force")}
    for _ in range(steps):
        root[0, 7:10] = root[0, 7:10] + g * dt
        root[0, 0:3] = root[0, 0:3] + root[0, 7:10] * dt
        hist["x"].append(root[0, 0:3].copy())
        hist["v_pre"].append(root[0, 7:10].copy())
        cts, cnt, _ = find_contacts(P, root[:, 0:3], [list(objects)])
        root, force, _ = solve(P, root, cts, cnt)
        hist["v"].append(root[0, 7:10].copy())
        hist["w"].append(root[0, 10:13].copy())
        hist["force"].append(force[0])
    return {k: np.asarray(a) for k, a in hist.items()}
