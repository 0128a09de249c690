"""Oracle of the rigid contact mode with dynamic obstacles (agx_hp2_contact_dynamic; DESIGN.md "Contact mode", "Dynamic obstacles").
TEST INFRASTRUCTURE ONLY.  Builds on oracle/contact_oracle.py (contact search, static solve):

* ``gather_bodies``: the bodies of each env's kept contacts, one per distinct asset in the order of its first contact.
* ``solve``: contact_core.cuh's two-body solve (contact_bodies_gather, contact_body_load, contact_solve_dynamic,
  contact_body_store) restated in numpy float32, vectorised over envs, every operation in the header's order, so it matches the
  kernel bit for bit given the same contact list.
* ``body_momentum`` / ``body_energy``: linear and angular momentum and kinetic energy of asset rows (float64), for the checks.
* ``simulate_dynamic``: a free sphere among free obstacles (no gravity on them), each sub-step in EnvManager's order (the obstacles
  drift, the sphere integrates, contacts are searched against the moved obstacles, the two-body solve writes them back)."""
import numpy as np

from .contact_oracle import CONTACT_MAX, _cross, _dot, _matvec, _where, find_contacts

f32 = np.float32


def gather_bodies(ids, count, obj_asset):
    """ids [E,CONTACT_MAX] (object index, K = ground), count [E], obj_asset [E,K] -> body [E,CONTACT_MAX] (index of the contact's
    body, -1 for the ground and unused slots), assets [E,CONTACT_MAX] (asset of each body, -1 unused), nb [E]"""
    ids, oa, count = np.asarray(ids), np.asarray(obj_asset), np.asarray(count)
    E, K = oa.shape
    body = np.full((E, CONTACT_MAX), -1, np.int64)
    assets = np.full((E, CONTACT_MAX), -1, np.int64)
    nb = np.zeros(E, np.int64)
    for e in range(E):
        for i in range(int(count[e])):
            if ids[e, i] >= K:
                continue
            a = int(oa[e, ids[e, i]])
            found = np.nonzero(assets[e, :nb[e]] == a)[0]
            if len(found):
                body[e, i] = found[0]
            else:
                assets[e, nb[e]], body[e, i] = a, nb[e]
                nb[e] += 1
    return body, assets, nb


def _quat_R(q):
    x, y, z, qw = q
    one, two = f32(1.0), f32(2.0)
    return [one - two * (y * y + z * z), two * (x * y - z * qw), two * (x * z + y * qw),
            two * (x * y + z * qw), one - two * (x * x + z * z), two * (y * z - x * qw),
            two * (x * z - y * qw), two * (y * z + x * qw), one - two * (x * x + y * y)]


def _world_inv_inertia(R, ii):
    A = [R[3 * i] * ii[j] + R[3 * i + 1] * ii[3 + j] + R[3 * i + 2] * ii[6 + j] for i in range(3) for j in range(3)]
    return [A[3 * i] * R[3 * j] + A[3 * i + 1] * R[3 * j + 1] + A[3 * i + 2] * R[3 * j + 2] for i in range(3) for j in range(3)]


def _keff(r, d, inv_m, Iw):
    rd = _cross(r, d)
    return inv_m + _dot(rd, _matvec(Iw, rd))


def _vel(v, w, r):
    wr = _cross(w, r)
    return [v[k] + wr[k] for k in range(3)]


def solve(P, root, contacts, count, ids, asset_state, obj_asset, mass):
    """root [E,>=13], contacts [E,CONTACT_MAX,7], count [E], ids [E,CONTACT_MAX], asset_state [E,A,>=13], obj_asset [E,K],
    mass [E,A,13] (inv_mass, com, inertia_inv) -> (root, force [E,3], crash [E], asset_state); inputs are not modified"""
    root = np.array(root, dtype=f32, copy=True)
    rows = np.array(asset_state, dtype=f32, copy=True)
    contacts = np.asarray(contacts, f32)
    mass = np.asarray(mass, f32)
    count = np.asarray(count)
    E = root.shape[0]
    ar = np.arange(E)
    body, assets, nb = gather_bodies(ids, count, obj_asset)
    # the bodies, per slot j: component arrays over envs (unused slots hold asset 0's values and are never used)
    S = range(CONTACT_MAX)
    Bx, Bq, Bv, Bw, Bc, Boc, Bm, BI, Bfree = ([] for _ in range(9))
    with np.errstate(all="ignore"):
        for j in S:
            a = np.maximum(assets[:, j], 0)
            row, m = rows[ar, a], mass[ar, a]
            x, q = [row[:, k] for k in range(3)], [row[:, 3 + k] for k in range(4)]
            R = _quat_R(q)
            cm = _matvec(R, [m[:, 1 + k] for k in range(3)])
            c = [x[k] + cm[k] for k in range(3)]
            Bx.append(x), Bq.append(q), Bv.append([row[:, 7 + k] for k in range(3)]), Bw.append([row[:, 10 + k] for k in range(3)])
            Bc.append(c), Boc.append([x[k] - c[k] for k in range(3)]), Bm.append(m[:, 0])
            BI.append(_world_inv_inertia(R, [m[:, 4 + k] for k in range(9)]))
            Bfree.append((m[:, 0] > 0) | (m[:, 4:13] != 0).any(axis=1))
    # the robot, as contact_solve
    ii, com_b = [f32(v) for v in P.inertia_inv], [f32(v) for v in P.com]
    rest, dt, maxd, mu = f32(P.rest_offset), f32(P.dt), f32(P.max_depenetration_velocity), f32(P.friction)
    R = _quat_R([root[:, 3 + k] for k in range(4)])
    com = _matvec(R, com_b)
    com = [root[:, k] + com[k] for k in range(3)]
    Iw = _world_inv_inertia(R, ii)
    zero = f32(0.0)
    inv_m = f32(1.0) / f32(P.mass)
    v = [root[:, 7 + k] for k in range(3)]
    w = [root[:, 10 + k] for k in range(3)]

    def apply(m, Pv, r, v, w):
        dw = _matvec(Iw, _cross(r, Pv))
        return _where(m, [v[k] + Pv[k] * inv_m for k in range(3)], v), _where(m, [w[k] + dw[k] for k in range(3)], w)

    def get(L, b):  # body b's values per env (b [E], >= 0)
        return [np.stack(L)[:, k][b, ar] for k in range(len(L[0]))] if isinstance(L[0], list) else np.stack(L)[b, ar]

    def body_apply(m, Pv, s, b):  # cbody_apply on body b of every env where m
        Iwb, ocb, imb = get(BI, b), get(Boc, b), get(Bm, b)
        dw = _matvec(Iwb, _cross(s, Pv))
        dwx = _cross(dw, ocb)
        vb, wb = get(Bv, b), get(Bw, b)
        nv = [vb[k] + (Pv[k] * imb + dwx[k]) for k in range(3)]
        nw = [wb[k] + dw[k] for k in range(3)]
        for k in range(3):
            for j in S:
                sel = m & (b == j)
                Bv[j][k] = np.where(sel, nv[k], Bv[j][k])
                Bw[j][k] = np.where(sel, nw[k], Bw[j][k])

    act = [count > i for i in S]
    hb = [body[:, i] >= 0 for i in S]
    bi = [np.maximum(body[:, i], 0) for i in S]
    nrm = [[contacts[:, i, 3 + k] for k in range(3)] for i in S]
    r = [[contacts[:, i, k] - com[k] for k in range(3)] for i in S]
    zeros = np.zeros(E, f32)
    with np.errstate(all="ignore"):
        ra = [[np.where(hb[i], contacts[:, i, k] - get(Bx, bi[i])[k], zero) for k in range(3)] for i in S]
        sa = [[np.where(hb[i], contacts[:, i, k] - get(Bc, bi[i])[k], zero) for k in range(3)] for i in S]
        kn = [np.where(hb[i], _keff(r[i], nrm[i], inv_m, Iw) + _keff(sa[i], nrm[i], get(Bm, bi[i]), get(BI, bi[i])),
                       _keff(r[i], nrm[i], inv_m, Iw)) for i in S]
        bias = [np.minimum(np.maximum(contacts[:, i, 6] - rest, zero) / dt, maxd) for i in S]
        ln = [zeros.copy() for _ in S]
        lt = [[zeros.copy() for _ in range(3)] for _ in S]

        def rel(i, v, w):
            vr = _vel(v, w, r[i])
            u = _vel(get(Bv, bi[i]), get(Bw, bi[i]), ra[i])
            return _where(hb[i], [vr[k] - u[k] for k in range(3)], vr)

        for _ in range(int(P.iterations)):
            for i in S:
                m, nn = act[i], nrm[i]
                pushes = m & hb[i] & get(Bfree, bi[i])
                vr = rel(i, v, w)
                dl = (bias[i] - _dot(nn, vr)) / kn[i]
                l1 = np.maximum(ln[i] + dl, zero)
                dl = l1 - ln[i]
                ln[i] = np.where(m, l1, ln[i])
                dP = [nn[k] * dl for k in range(3)]
                v, w = apply(m, dP, r[i], v, w)
                body_apply(pushes, [-dP[k] for k in range(3)], sa[i], bi[i])
                vr = rel(i, v, w)
                vn = _dot(nn, vr)
                vt = [vr[k] - nn[k] * vn for k in range(3)]
                s = np.sqrt(_dot(vt, vt))
                t = [vt[k] / s for k in range(3)]
                kt = _keff(r[i], t, inv_m, Iw)
                kt = np.where(hb[i], kt + _keff(sa[i], t, get(Bm, bi[i]), get(BI, bi[i])), kt)
                dt_ = s / kt
                l2 = _where(s > zero, [lt[i][k] - t[k] * dt_ for k in range(3)], lt[i])
                mag, lim = np.sqrt(_dot(l2, l2)), mu * ln[i]
                f = lim / mag
                l2 = _where(mag > lim, [l2[k] * f for k in range(3)], l2)
                dP = [l2[k] - lt[i][k] for k in range(3)]
                lt[i] = _where(m, l2, lt[i])
                v, w = apply(m, dP, r[i], v, w)
                body_apply(pushes, [-dP[k] for k in range(3)], sa[i], bi[i])
        # contact_body_store
        half = f32(0.5)
        for j in S:
            wr = (j < nb) & Bfree[j]
            a = np.maximum(assets[:, j], 0)
            row = rows[ar, a]
            q = Bq[j]
            xn = [Bx[j][k] + (Bv[j][k] - row[:, 7 + k]) * dt for k in range(3)]
            h = [(Bw[j][k] - row[:, 10 + k]) * dt * half for k in range(3)]
            qn = [q[0] + h[0] * q[3] + h[1] * q[2] - h[2] * q[1],
                  q[1] - h[0] * q[2] + h[1] * q[3] + h[2] * q[0],
                  q[2] + h[0] * q[1] - h[1] * q[0] + h[2] * q[3],
                  q[3] - h[0] * q[0] - h[1] * q[1] - h[2] * q[2]]
            inv = f32(1.0) / np.sqrt(qn[0] * qn[0] + qn[1] * qn[1] + qn[2] * qn[2] + qn[3] * qn[3])
            new = row.copy()
            for k in range(3):
                new[:, k] = xn[k]
                new[:, 7 + k] = Bv[j][k]
                new[:, 10 + k] = Bw[j][k]
            for k in range(4):
                new[:, 3 + k] = qn[k] * inv
            rows[ar[wr], a[wr]] = new[wr]
    imp = [zeros.copy() for _ in range(3)]
    for i in S:
        imp = _where(act[i], [imp[k] + nrm[i][k] * ln[i] + lt[i][k] for k in range(3)], imp)
    force = np.stack([imp[k] / dt for k in range(3)], axis=1)
    crash = (count > 0) & (np.sqrt(_dot([force[:, 0], force[:, 1], force[:, 2]], [force[:, 0], force[:, 1], force[:, 2]])) > f32(P.force_threshold))
    force[count == 0] = 0.0
    for k in range(3):
        root[:, 7 + k] = v[k]
        root[:, 10 + k] = w[k]
    return root, force, crash, rows


def _R64(q):
    x, y, z, w = (float(c) for c in q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def _com_velocity(row, com, origin_twist):
    row = np.asarray(row, np.float64)
    R = _R64(row[3:7])
    c = row[0:3] + R @ np.asarray(com, np.float64)
    w = row[10:13]
    vc = row[7:10] + np.cross(w, c - row[0:3]) if origin_twist else row[7:10]
    return R, c, w, vc


def body_momentum(row, mass, com, inertia, about=(0.0, 0.0, 0.0), origin_twist=True):
    """(linear, angular about `about`) momentum of a rigid body in float64 from its row, its mass, COM (body frame) and inertia
    about the COM (body frame).  origin_twist: the row's v is the velocity of its origin (an asset row); False: of its COM (the
    robot's root state as the contact solve treats it)"""
    R, c, w, vc = _com_velocity(row, com, origin_twist)
    p = mass * vc
    L = np.cross(c - np.asarray(about, np.float64), p) + R @ np.asarray(inertia, np.float64) @ R.T @ w
    return p, L


def body_energy(row, mass, com, inertia, origin_twist=True):
    """kinetic energy in float64, arguments as body_momentum's"""
    R, c, w, vc = _com_velocity(row, com, origin_twist)
    return 0.5 * mass * vc @ vc + 0.5 * w @ (R @ np.asarray(inertia, np.float64) @ R.T @ w)


def robot_row_body(P):
    """(mass, com, inertia) of the robot described by P, for body_momentum / body_energy"""
    return float(P.mass), np.array(list(P.com), np.float64), np.linalg.inv(np.array(list(P.inertia_inv), np.float64).reshape(3, 3))


def simulate_dynamic(P, x, v, w, steps, bodies, gravity=(0.0, 0.0, 0.0)):
    """a free sphere (robot of P) among free obstacles.  bodies: list of dicts with "tris" ([n,9] triangles a, ab, ac in the body
    frame), "x" (origin), optional "q" (x y z w), "v", "w" (twist of the origin), "mass", "com" (body frame), "inertia" (about the
    COM, body frame).  Per sub-step: each body drifts (x += v dt, q = normalize(dq(w dt) (x) q), float32, no damping), the sphere
    integrates (v += g dt, x += v dt), contacts are searched against the moved bodies (no ground), and the two-body solve runs
    and writes the bodies back.  Returns per sub-step: robot root row, body rows [B,13], force."""
    root = np.zeros((1, 13), f32)
    root[0, 0:3], root[0, 6], root[0, 7:10], root[0, 10:13] = x, 1.0, v, w
    g, dt = np.asarray(gravity, f32), f32(P.dt)
    B = len(bodies)
    rows = np.zeros((1, B, 13), f32)
    mass = np.zeros((1, B, 13), f32)
    for j, b in enumerate(bodies):
        rows[0, j, 0:3], rows[0, j, 3:7] = b["x"], b.get("q", (0.0, 0.0, 0.0, 1.0))
        rows[0, j, 7:10], rows[0, j, 10:13] = b.get("v", (0, 0, 0)), b.get("w", (0, 0, 0))
        mass[0, j, 0], mass[0, j, 1:4] = 1.0 / b["mass"], b.get("com", (0, 0, 0))
        mass[0, j, 4:13] = np.linalg.inv(np.asarray(b["inertia"], np.float64)).reshape(9)
    tris = [np.asarray(b["tris"], np.float64).reshape(-1, 3, 3) for b in bodies]
    obj_asset = np.arange(B, dtype=np.int32)[None]
    hist = {k: [] for k in ("root", "rows", "force")}
    half = f32(0.5)
    for _ in range(steps):
        for j in range(B):
            r = rows[0, j]
            r[0:3] = r[0:3] + r[7:10] * dt
            h = r[10:13] * dt * half
            q = r[3:7].copy()
            qn = np.array([q[0] + h[0] * q[3] + h[1] * q[2] - h[2] * q[1], q[1] - h[0] * q[2] + h[1] * q[3] + h[2] * q[0],
                           q[2] + h[0] * q[1] - h[1] * q[0] + h[2] * q[3], q[3] - h[0] * q[0] - h[1] * q[1] - h[2] * q[2]], f32)
            r[3:7] = qn / np.sqrt((qn * qn).sum())
        root[0, 7:10] = root[0, 7:10] + g * dt
        root[0, 0:3] = root[0, 0:3] + root[0, 7:10] * dt
        world = []
        for j in range(B):
            R = _R64(rows[0, j, 3:7])
            t = tris[j]
            world.append(np.concatenate([t[:, 0] @ R.T + rows[0, j, 0:3], t[:, 1] @ R.T, t[:, 2] @ R.T], axis=1).astype(f32))
        cts, cnt, ids = find_contacts(P, root[:, 0:3], [world])
        root, force, _, rows = solve(P, root, cts, cnt, ids, rows, obj_asset, mass)
        hist["root"].append(root[0].copy())
        hist["rows"].append(rows[0].copy())
        hist["force"].append(force[0])
    return {k: np.asarray(a) for k, a in hist.items()}
