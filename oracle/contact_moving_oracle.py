"""Oracle of the rigid contact mode with moving obstacles (agx_hp2_contact_moving; DESIGN.md "Contact mode", "Moving obstacles").
TEST INFRASTRUCTURE ONLY.  Builds on oracle/contact_oracle.py (contact search, static solve):

* ``solve(..., obstacle_velocity=u)``: contact_core.cuh's MOVING solve restated in numpy float32 in the header's operation order:
  both rows act on v_robot(p) - u.  ``obstacle_velocity=None`` is contact_oracle.solve itself.
* ``obstacle_point_velocity``: u from the asset rows and the contact ids, in the kernel's order.
* ``simulate_moving``: a free sphere among obstacles that move with a twist, each sub-step in EnvManager's order (obstacles, then
  the sphere's integration, the contact search and the solve), for the physical checks."""
import numpy as np

from .contact_oracle import CONTACT_MAX, _cross, _dot, _matvec, _where, closest_points, find_contacts
from .contact_oracle import solve as static_solve

f32 = np.float32


def solve(P, root, contacts, count, obstacle_velocity=None):
    """root [E,>=13] float32 (copied), contacts [E,CONTACT_MAX,7] (point, normal, depth), count [E], obstacle_velocity
    [E,CONTACT_MAX,3] (each contact's obstacle velocity at its point) -> (root, force [E,3], crash [E])"""
    if obstacle_velocity is None:
        return static_solve(P, root, contacts, count)
    root = np.array(root, dtype=f32, copy=True)
    contacts = np.asarray(contacts, f32)
    uo = np.asarray(obstacle_velocity, f32)
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

    def rel_vel(v, w, r, u):  # cvel, then minus the obstacle's velocity
        wr = _cross(w, r)
        vr = [v[k] + wr[k] for k in range(3)]
        return [vr[k] - u[k] for k in range(3)]

    S = range(CONTACT_MAX)
    act = [count > i for i in S]
    nrm = [[contacts[:, i, 3 + k] for k in range(3)] for i in S]
    u = [[uo[:, i, k] for k in range(3)] for i in S]
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
                vr = rel_vel(v, w, r[i], u[i])
                dl = (bias[i] - _dot(nn, vr)) / kn[i]
                l1 = np.maximum(ln[i] + dl, zero)
                dl = l1 - ln[i]
                ln[i] = np.where(m, l1, ln[i])
                v, w = apply(m, [nn[k] * dl for k in range(3)], r[i], v, w)
                vr = rel_vel(v, w, r[i], u[i])
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


def obstacle_point_velocity(asset_state, obj_asset, contacts, ids):
    """u [E,CONTACT_MAX,3] float32 as the kernel computes it: for a contact with object k of env e, the row of asset
    a = obj_asset[e,k] (x y z q v w) gives u = v + w x (p - x), in contact_core.cuh's order; the ground (id = K) and unused slots
    (-1) get 0"""
    st = np.asarray(asset_state, f32)
    oa = np.asarray(obj_asset)
    cts = np.asarray(contacts, f32)
    ids = np.asarray(ids)
    E, K = oa.shape
    u = np.zeros((E, CONTACT_MAX, 3), f32)
    for e in range(E):
        for i in range(CONTACT_MAX):
            k = int(ids[e, i])
            if 0 <= k < K:
                row = st[e, oa[e, k]]
                r = [cts[e, i, j] - row[j] for j in range(3)]
                wr = _cross(row[10:13], r)
                u[e, i] = [row[7 + j] + wr[j] for j in range(3)]
    return u


def simulate_moving(P, x, v, w, steps, bodies, gravity=(0.0, 0.0, -9.81)):
    """contact_oracle.simulate among moving obstacles.  bodies: list of dicts with "tris" ([n,9] triangles a, ab, ac in the body
    frame), "x" (body origin, world), "v" (linear velocity) and "wz" (angular velocity about the world z axis through the origin).
    Per sub-step, in EnvManager's order with args['contact_moving_obstacles']: every body advances by dt (x += v dt, yaw += wz dt,
    float64), the sphere integrates (v += g dt, x += v dt), contacts are searched against the moved bodies and the ground, and the
    solve runs with each contact's body velocity u = v + w x (p - x).  Returns per sub-step: x, v_pre (after the integration), v, w
    (after the solve), force, and depth (the deepest penetration radius - distance into any body, after the integration)."""
    root = np.zeros((1, 13), f32)
    root[0, 0:3], root[0, 6], root[0, 7:10], root[0, 10:13] = x, 1.0, v, w
    g, dt = np.asarray(gravity, f32), f32(P.dt)
    st = [dict(x=np.asarray(b["x"], np.float64), v=np.asarray(b["v"], np.float64), wz=float(b.get("wz", 0.0)), yaw=0.0,
               tris=np.asarray(b["tris"], np.float64).reshape(-1, 3, 3)) for b in bodies]
    hist = {k: [] for k in ("x", "v_pre", "v", "w", "force", "depth")}
    for _ in range(steps):
        world, rows = [], np.zeros((1, len(st), 13), f32)
        for j, b in enumerate(st):
            b["x"] = b["x"] + b["v"] * float(dt)
            b["yaw"] += b["wz"] * float(dt)
            c, s = np.cos(b["yaw"]), np.sin(b["yaw"])
            R = np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])
            t = b["tris"]
            world.append(np.concatenate([t[:, 0] @ R.T + b["x"], t[:, 1] @ R.T, t[:, 2] @ R.T], axis=1).astype(f32))
            rows[0, j, 0:3], rows[0, j, 6], rows[0, j, 7:10], rows[0, j, 12] = b["x"], 1.0, b["v"], b["wz"]
        root[0, 7:10] = root[0, 7:10] + g * dt
        root[0, 0:3] = root[0, 0:3] + root[0, 7:10] * dt
        hist["x"].append(root[0, 0:3].copy())
        hist["v_pre"].append(root[0, 7:10].copy())
        hist["depth"].append(max([float(P.radius) - float(np.sqrt(closest_points(root[0, 0:3], tr)[1].min())) for tr in world]
                                 + [-np.inf]))
        cts, cnt, ids = find_contacts(P, root[:, 0:3], [world])
        u = obstacle_point_velocity(rows, np.arange(len(st), dtype=np.int32)[None], cts, ids)
        root, force, _ = solve(P, root, cts, cnt, obstacle_velocity=u)
        hist["v"].append(root[0, 7:10].copy())
        hist["w"].append(root[0, 10:13].copy())
        hist["force"].append(force[0])
    return {k: np.asarray(a) for k, a in hist.items()}
