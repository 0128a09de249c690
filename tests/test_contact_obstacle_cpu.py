"""Contact between free obstacles on the CPU: contact_core.cuh's box-box narrow phase and two-body solve (compiled for the host)
against oracle/contact_obstacle_oracle.py bit for bit, the separating-axis depth and normal against a float64 brute force, the
physics cases (head-on cubes, a cube resting on a plate, crossed plates, an off-centre hit, Coulomb friction, energy, untouched
rows, a dynamic_env reset pulled apart), the argument checks and an end-to-end dynamic_env run on the CPU stack."""
import ctypes as C
import random

import numpy as np
import pytest
import torch

from aerial_gym_simulator_b200 import _lib
from aerial_gym_simulator_b200.hp2 import ObstacleBoxes, box_obb
from oracle import contact_dynamic_oracle as CD
from oracle import contact_obstacle_oracle as CO
from tests._cpu_stack_obstacle_contact import ground_shadow, obstacle_obstacle_shadow, obstacle_twins
from tests.test_contact_cpu import params

# the four box files of environment_assets/objects (dynamic_env), and one box off-centre and turned in its asset frame
SIZES = [(0.1, 0.1, 2.0), (0.1, 0.5, 0.5), (0.1, 1.0, 1.0), (0.4, 0.4, 0.4)]


def _rot(axis, ang):
    a = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(ang) * K + (1 - np.cos(ang)) * K @ K


def _quat(R):
    from aerial_gym_simulator_b200.env_manager.env_manager import _matrix_to_quat
    return _matrix_to_quat(np.asarray(R, np.float64))


def _boxes():
    rows = [box_obb(s)[:15] for s in SIZES] + [box_obb((0.3, 0.2, 0.6), _rot((1, 2, 3), 0.7), (0.1, -0.05, 0.2))[:15]]
    return np.stack(rows).astype(np.float32)


def _box_mass(m, size, com=(0.0, 0.0, 0.0)):
    J = np.diag([size[1] ** 2 + size[2] ** 2, size[0] ** 2 + size[2] ** 2, size[0] ** 2 + size[1] ** 2]) * m / 12.0
    return np.concatenate([[1.0 / m], com, np.linalg.inv(J).reshape(9)]).astype(np.float32)


def _params(**kw):
    d = dict(contact_offset=0.002, rest_offset=0.001, dt=0.01, friction=1.0, max_depenetration_velocity=1.0, iterations=4)
    d.update(kw)
    return params(**d)


def random_envs(E, A, seed, spread=1.2, kinematic=0.15, vscale=2.0):
    """E envs of A boxes (random files) in a cube of side `spread`, random orientations, |v| <= vscale, |w| <= 2; masses 0.2-5 kg
    with a COM up to 0.1 m off the origin and the box inertia, a `kinematic` fraction of all-zero rows"""
    g = np.random.default_rng(seed)
    rows = np.zeros((E, A, 13), np.float32)
    rows[..., 0:3] = g.uniform(-spread / 2, spread / 2, (E, A, 3))
    q = g.normal(size=(E, A, 4))
    rows[..., 3:7] = q / np.linalg.norm(q, axis=-1, keepdims=True)
    d = g.normal(size=(E, A, 6))
    rows[..., 7:10] = d[..., 0:3] / np.linalg.norm(d[..., 0:3], axis=-1, keepdims=True) * g.uniform(0, vscale, (E, A, 1))
    rows[..., 10:13] = d[..., 3:6] / np.linalg.norm(d[..., 3:6], axis=-1, keepdims=True) * g.uniform(0, 2, (E, A, 1))
    boxes = _boxes()
    af = g.integers(0, len(boxes), (E, A)).astype(np.int32)
    mass = np.zeros((E, A, 13), np.float32)
    for e in range(E):
        for a in range(A):
            mass[e, a] = _box_mass(g.uniform(0.2, 5.0), boxes[af[e, a], 12:15] * 2, g.uniform(-0.1, 0.1, 3))
    mass[g.uniform(size=(E, A)) < kinematic] = 0.0
    return rows, mass, boxes, af


def shadow(P, rows, mass, boxes, af):
    r = np.ascontiguousarray(rows, np.float32).copy()
    count, contacts = obstacle_obstacle_shadow(P, r, mass, boxes, af)
    return r, count, contacts


def oracle(P, rows, mass, boxes, af):
    out, lists, kinds = np.zeros_like(rows), [], {}
    for e in range(rows.shape[0]):
        out[e], L, k = CO.env_contact(P, rows[e], mass[e], boxes, af[e])
        lists.append(L)
        kinds.update({(e,) + key: v for key, v in k.items()})
    return out, lists, kinds


def _same_list(count, contacts, lists):
    for e, L in enumerate(lists):
        assert count[e] == len(L), (e, count[e], len(L))
        for q, (p, n, dep, i, j) in enumerate(L):
            ref = np.array([*p, *n, dep, i, j], np.float32)
            assert np.array_equal(contacts[e, q], ref), (e, q, contacts[e, q], ref)


@pytest.mark.parametrize("iterations,friction,seed", [(1, 0.0, 0), (4, 1.0, 1), (10, 0.5, 2), (4, 2.0, 3)])
def test_shadow_matches_oracle_bit_for_bit_on_piles(iterations, friction, seed):
    P = _params(iterations=iterations, friction=friction)
    rows, mass, boxes, af = random_envs(10, 10, seed)
    got, count, contacts = shadow(P, rows, mass, boxes, af)
    ref, lists, kinds = oracle(P, rows, mass, boxes, af)
    _same_list(count, contacts, lists)
    assert np.array_equal(got, ref), f"{(got != ref).any(-1).sum()} rows differ"
    assert {"faceA", "faceB", "edge"} <= set(kinds.values()) and count.max() >= 8 and count.sum() > 40


@pytest.mark.parametrize("iterations,friction,seed", [(4, 1.0, 11), (10, 0.3, 12)])
def test_shadow_matches_oracle_bit_for_bit_on_pairs(iterations, friction, seed):
    """one pair per env, placed so that about half touch"""
    P = _params(iterations=iterations, friction=friction)
    rows, mass, boxes, af = random_envs(400, 2, seed, spread=0.9, kinematic=0.1)
    got, count, contacts = shadow(P, rows, mass, boxes, af)
    ref, lists, kinds = oracle(P, rows, mass, boxes, af)
    _same_list(count, contacts, lists)
    assert np.array_equal(got, ref), f"{(got != ref).any(-1).sum()} rows differ"
    touched = count > 0
    assert 0.2 < touched.mean() < 0.9 and not (got[~touched] != rows[~touched]).any()
    assert sum(v == "edge" for v in kinds.values()) > 5


def _world_boxes(row, box):
    b = CO.box_world(np.asarray(row, np.float32), box)
    return np.array(b["c"], np.float64), np.array(b["a"], np.float64), np.array(b["h"], np.float64)


def _support(c, ax, h, n):
    return c @ n + np.abs(ax @ n) @ h


def test_sat_depth_and_normal_against_brute_force_float64():
    """the contact normal is the direction of least overlap: no sampled direction separates the boxes with less, the chosen
    axis' overlap equals the manifold's depth, and every face contact's incident point lies inside the reference box with the
    signed distance the manifold gives (surface samples of the incident box, float64)"""
    P = _params()
    rows, mass, boxes, af = random_envs(600, 2, 21, spread=0.8, kinematic=0.0)
    g = np.random.default_rng(22)
    dirs = g.normal(size=(4000, 3))
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    checked = {"faceA": 0, "faceB": 0, "edge": 0}
    for e in range(rows.shape[0]):
        A, B = (CO.box_world(rows[e, k], boxes[af[e, k]]) for k in (0, 1))
        c, kind = CO.box_pair(P, A, B)
        if not c:
            continue
        (ca, aa, ha), (cb, ab, hb) = _world_boxes(rows[e, 0], boxes[af[e, 0]]), _world_boxes(rows[e, 1], boxes[af[e, 1]])
        n = np.array(c[0][1], np.float64)
        overlap = lambda u: _support(ca, aa, ha, u) + _support(cb, ab, hb, -u)  # max over A of x.u - min over B of y.u
        depth = overlap(n)
        best = min(overlap(u) for u in np.concatenate([dirs, -dirs]))
        tol = 2e-5 * (1.0 + np.abs(ca).max() + np.abs(cb).max())
        axes = [*aa, *ab] + [np.cross(x, y) for x in aa for y in ab if np.linalg.norm(np.cross(x, y)) > 1e-3]
        m15 = min(min(overlap(u / np.linalg.norm(u)), overlap(-u / np.linalg.norm(u))) for u in axes)
        assert m15 <= best + tol, (e, m15, best)  # the 15 axes hold the least overlap of any direction
        assert m15 - tol <= depth <= m15 + 2 * 1e-4 + tol, (e, kind, depth, m15)  # the chosen axis, within the stated bias
        if kind == "edge":
            assert abs(c[0][2] - depth) <= tol, (e, c[0][2], depth)
        else:
            (cr, ar, hr) = (ca, aa, ha) if kind == "faceA" else (cb, ab, hb)
            nr = n if kind == "faceA" else -n
            for p, _, dep in c:
                if dep > 2.0 * hr.min():
                    continue  # deeper than the reference box is thick: the incident point is out through its far side
                x = np.array(p, np.float64) - nr * float(dep) / 2.0  # the incident point
                sd = CO.box_signed_distance(x[None], cr, ar, hr)[0]
                assert sd >= -float(dep) - tol and (dep <= 0 or sd <= tol), (e, kind, sd, dep)
            assert max(float(x[2]) for x in c) <= depth + tol
        checked[kind] += 1
    assert min(checked.values()) >= 10, checked


def _pair(P, rowA, rowB, boxA, boxB, mA, mB):
    rows = np.stack([rowA, rowB]).astype(np.float32)[None]
    mass = np.stack([mA, mB]).astype(np.float32)[None]
    boxes = np.stack([boxA, boxB]).astype(np.float32)
    af = np.array([[0, 1]], np.int32)
    got, count, contacts = shadow(P, rows, mass, boxes, af)
    ref, lists, kinds = oracle(P, rows, mass, boxes, af)
    assert np.array_equal(got, ref)
    _same_list(count, contacts, lists)
    return got[0], lists[0], kinds.get((0, 0, 1), "none")


def _row(x, R=np.eye(3), v=(0.0, 0.0, 0.0), w=(0.0, 0.0, 0.0)):
    return np.concatenate([x, _quat(R), v, w]).astype(np.float32)


def _momentum(rows, masses):
    """(linear, angular about the origin) momentum of asset rows with box mass rows, float64"""
    lin, ang = np.zeros(3), np.zeros(3)
    for r, m in zip(rows, masses):
        R, c, w, vc = CD._com_velocity(r, m[1:4].astype(np.float64), True)
        M = 1.0 / float(m[0])
        J = R @ np.linalg.inv(m[4:13].astype(np.float64).reshape(3, 3)) @ R.T
        lin += M * vc
        ang += np.cross(c, M * vc) + J @ w
    return lin, ang


def _energy(rows, masses):
    return sum(CD.body_energy(r, 1.0 / float(m[0]), m[1:4], np.linalg.inv(m[4:13].astype(np.float64).reshape(3, 3)))
               for r, m in zip(rows, masses))


@pytest.mark.parametrize("friction", [0.0, 1.0])
def test_head_on_equal_cubes_stop_relative_motion_and_conserve_momentum(friction):
    P = _params(iterations=10, friction=friction)
    cube = box_obb((0.4, 0.4, 0.4))[:15]
    m = _box_mass(1.0, (0.4, 0.4, 0.4))
    a = _row((-0.2 + 0.00025, 0.03, 0.0), v=(1.0, 0.0, 0.0))
    b = _row((0.2 - 0.00025, -0.03, 0.0), v=(-1.0, 0.0, 0.0))  # 0.5 mm deep: below rest_offset, no bias
    got, L, kind = _pair(P, a, b, cube, cube, m, m)
    assert kind == "faceA" and len(L) == 4
    # zero relative normal velocity at every contact point (the cubes are off-centre, so they also spin)
    vel = lambda r, p: r[7:10].astype(np.float64) + np.cross(r[10:13].astype(np.float64), np.asarray(p, np.float64) - r[0:3])
    vn = [float(np.dot(n, vel(got[1], p) - vel(got[0], p))) for p, n, *_ in L]
    assert np.abs(vn).max() <= 1e-3, vn  # 0.05 % of the approach speed: what the iterations leave with the cubes spinning
    assert np.abs(got[:, 10:13]).max() > 0.1
    l0, h0 = _momentum([a, b], [m, m])
    after = np.stack([a, b])
    after[:, 7:13] = got[:, 7:13]  # the solve's twists on the poses it ran with
    l1, h1 = _momentum(after, [m, m])
    assert np.abs(l1 - l0).max() <= 4 * 2 ** -23 * 2.0 and np.abs(h1 - h0).max() <= 4 * 2 ** -23 * 2.0, (l1 - l0, h1 - h0)


def test_a_cube_resting_face_down_on_a_plate_gets_four_contacts():
    P = _params()
    plate, cube = box_obb((0.1, 1.0, 1.0))[:15], box_obb((0.4, 0.4, 0.4))[:15]
    lay = _rot((0, 1, 0), np.pi / 2)  # the plate's thin x axis vertical
    a = _row((0.0, 0.0, 0.0), lay)
    b = _row((0.1, -0.15, 0.05 + 0.2 - 0.0005), v=(0.0, 0.0, -0.5))
    got, L, kind = _pair(P, a, b, plate, cube, _box_mass(2.0, (0.1, 1, 1)), _box_mass(1.0, (0.4, 0.4, 0.4)))
    assert len(L) == 4 and kind in ("faceA", "faceB")
    nz = np.array([x[1] for x in L])
    assert np.allclose(nz, [0.0, 0.0, 1.0], atol=1e-6)
    assert got[1, 9] > -0.5 and got[0, 9] < 0.0  # the cube slows, the plate is pushed down


def test_two_plates_crossed_in_an_x_touch_edge_to_edge_and_are_pushed_apart():
    """plate A's top edge (along x) under plate B's bottom edge (along y), each plate turned 45 degrees about its edge so that the
    edge is its extreme line: no vertex of either is inside the other, only the edges cross"""
    P = _params(friction=0.5)
    plate = box_obb((0.1, 1.0, 1.0))[:15]  # half extents 0.05, 0.5, 0.5
    depth = 0.004
    Ra = _rot((1, 0, 0), np.pi / 4) @ _rot((0, 0, 1), np.pi / 2)   # thin axis along y, then 45 deg about x
    Rb = _rot((0, 1, 0), np.pi / 4)                                  # thin axis along x, 45 deg about y
    ext = lambda R: float(np.abs(R @ np.diag([0.05, 0.5, 0.5])).sum(axis=1)[2])  # the box's half height
    a = _row((0.0, 0.0, -ext(Ra) + depth / 2), Ra)
    b = _row((0.0, 0.0, ext(Rb) - depth / 2), Rb)
    m = _box_mass(1.0, (0.1, 1.0, 1.0))
    got, L, kind = _pair(P, a, b, plate, plate, m, m)
    assert kind == "edge" and len(L) == 1
    p, n, dep, *_ = L[0]
    # at the crossing of A's top edge and B's bottom edge
    corners = np.array([[sx, sy, sz] for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)]) * np.array([0.05, 0.5, 0.5])
    top = (corners @ Ra.T + a[0:3])[np.argsort(-(corners @ Ra.T)[:, 2])[:2]]
    bottom = (corners @ Rb.T + b[0:3])[np.argsort((corners @ Rb.T)[:, 2])[:2]]
    assert np.ptp(top[:, 1]) < 1e-9 and np.ptp(bottom[:, 0]) < 1e-9  # the edges run along x and along y
    assert np.allclose(n, [0.0, 0.0, 1.0], atol=1e-5) and abs(dep - depth) < 2e-5
    assert abs(p[0] - bottom[0, 0]) < 1e-4 and abs(p[1] - top[0, 1]) < 1e-4 and abs(p[2] - (top[0, 2] + bottom[0, 2]) / 2) < 1e-4
    # pushed apart: B up, A down, the contact point separating at the depenetration target (depth - rest_offset) / dt
    vel = lambda r: r[7:10].astype(np.float64) + np.cross(r[10:13].astype(np.float64), np.asarray(p, np.float64) - r[0:3])
    assert got[1, 9] > 0.0 > got[0, 9]
    assert abs((vel(got[1]) - vel(got[0]))[2] - (dep - P.rest_offset) / P.dt) < 1e-3


def test_an_off_centre_rod_hit_spins_the_cube_by_its_lever_arm():
    P = _params(friction=0.0, iterations=10)
    rod, cube = box_obb((0.1, 0.1, 2.0))[:15], box_obb((0.4, 0.4, 0.4))[:15]
    mr, mc = _box_mass(3.0, (0.1, 0.1, 2.0)), _box_mass(1.0, (0.4, 0.4, 0.4))
    for y in (0.12, -0.08):
        a = _row((-0.25 + 0.0005, y, 0.0), v=(2.0, 0.0, 0.0))   # the rod, standing, moving +x
        b = _row((0.0, 0.0, 0.0))                                # the cube at rest
        got, L, _ = _pair(P, a, b, rod, cube, mr, mc)
        assert len(L) == 4
        dv, dw = float(got[1, 7]), float(got[1, 12])
        Izz = 1.0 / float(mc[12])
        # dw_z = -(lever arm) m dv_x / I_zz, the lever arm between the rod's two faces y -+ 0.05
        assert dv > 0 and np.sign(dw) == -np.sign(y)
        arm = -dw * Izz / (1.0 * dv)
        assert min(y - 0.05, y + 0.05) - 1e-4 <= arm <= max(y - 0.05, y + 0.05) + 1e-4, (y, arm)


@pytest.mark.parametrize("mu", [0.0, 1.0])
def test_an_oblique_impact_obeys_coulomb(mu):
    P = _params(friction=mu, iterations=10)
    cube = box_obb((0.4, 0.4, 0.4))[:15]
    m = _box_mass(1.0, (0.4, 0.4, 0.4))
    g = np.random.default_rng(30)
    for _ in range(20):
        vt = g.uniform(-3, 3, 2)
        a = _row((0.0, 0.0, 0.0), w=g.normal(size=3) * 0.3)
        b = _row((0.0, g.uniform(-0.1, 0.1), 0.4 - 0.0005), v=(vt[0], vt[1], -g.uniform(0.5, 3)))
        got, L, _ = _pair(P, a, b, cube, cube, m, m)
        assert len(L) == 4
        _, _, _, vb0 = CD._com_velocity(b, m[1:4].astype(np.float64), True)
        _, _, _, vb1 = CD._com_velocity(got[1], m[1:4].astype(np.float64), True)
        dp = vb1 - vb0  # impulse on B per unit mass (1 kg)
        assert dp[2] > 0 and np.linalg.norm(dp[0:2]) <= mu * dp[2] * (1 + 1e-5) + 1e-6, (dp, mu)


def test_kinetic_energy_never_rises_without_bias():
    rows, mass, boxes, af = random_envs(60, 8, 31, kinematic=0.0)
    for friction in (0.0, 0.5, 2.0):
        P = _params(friction=friction, rest_offset=10.0, contact_offset=0.01)  # every depth below rest_offset: no bias
        got, count, contacts = shadow(P, rows, mass, boxes, af)
        checked = 0
        for e in np.nonzero(count)[0]:
            after = rows[e].copy()
            after[:, 7:13] = got[e, :, 7:13]  # the solve's twists on the poses it ran with
            e0, e1 = _energy(rows[e], mass[e]), _energy(after, mass[e])
            assert e1 <= e0 * (1 + 1e-5) + 1e-6, (friction, e, e0, e1)
            checked += 1
        assert checked > 30


def test_boxes_beyond_contact_offset_and_kinematic_rows_are_untouched():
    P = _params()
    cube = box_obb((0.4, 0.4, 0.4))[:15]
    m = _box_mass(1.0, (0.4, 0.4, 0.4))
    for gap in (P.contact_offset * 1.01, 0.01, 1.0):
        a, b = _row((0.0, 0.0, 0.0), v=(1.0, 0, 0)), _row((0.4 + gap, 0.0, 0.0), v=(-1.0, 0, 0))
        got, L, _ = _pair(P, a, b, cube, cube, m, m)
        assert not L and np.array_equal(got, np.stack([a, b]))
    # within contact_offset but not penetrating: a contact, no bias, the approach is stopped
    a, b = _row((0.0, 0.0, 0.0), v=(1.0, 0, 0)), _row((0.4 + P.contact_offset * 0.5, 0.0, 0.0), v=(-1.0, 0, 0))
    got, L, _ = _pair(P, a, b, cube, cube, m, m)
    assert len(L) == 4 and got[1, 7] - got[0, 7] > -1e-5
    # kinematic rows: read, never written; two kinematic rows are not a pair
    rows, mass, boxes, af = random_envs(30, 10, 32, kinematic=0.5)
    got, count, contacts = shadow(P, rows, mass, boxes, af)
    kin = ~mass.any(-1)
    assert np.array_equal(got[kin], rows[kin]) and count.sum() > 20
    for e in range(30):
        for q in range(count[e]):
            i, j = int(contacts[e, q, 7]), int(contacts[e, q, 8])
            assert not (kin[e, i] and kin[e, j])
    moved_by_kinematic = False
    for e in range(30):
        for q in range(count[e]):
            i, j = int(contacts[e, q, 7]), int(contacts[e, q, 8])
            moved_by_kinematic |= bool(kin[e, i] != kin[e, j])
    assert moved_by_kinematic


def test_the_list_keeps_whole_pairs_in_order_until_it_is_full():
    """a stack of coincident boxes (parked assets) fills the list: pairs go in (i, j) order until one no longer fits"""
    P = _params()
    E, A = 1, 20
    rows = np.zeros((E, A, 13), np.float32)
    rows[..., 0:3] = -1000.0
    rows[..., 6] = 1.0
    boxes = np.stack([box_obb((0.4, 0.4, 0.4))[:15]])
    mass = np.broadcast_to(_box_mass(1.0, (0.4, 0.4, 0.4)), (E, A, 13)).copy()
    af = np.zeros((E, A), np.int32)
    got, count, contacts = shadow(P, rows, mass, boxes, af)
    ref, lists, _ = oracle(P, rows, mass, boxes, af)
    _same_list(count, contacts, lists)
    assert np.array_equal(got, ref)
    pairs = [(int(contacts[0, q, 7]), int(contacts[0, q, 8])) for q in range(count[0])]
    assert count[0] == 128 and pairs == sorted(pairs) and pairs[0] == (0, 1) and len(set(pairs)) == 32


def _dynamic_env(n, seed=0, env_name="dynamic_env", **extra):
    from aerial_gym_simulator_b200.env_manager import EnvManager
    args = {"contact": "rigid", "contact_moving_obstacles": True, "contact_dynamic_obstacles": True, "contact_obstacle_obstacle": True,
            "seed": seed, **extra}
    random.seed(seed)
    torch.manual_seed(seed)
    return EnvManager("base_sim", env_name, "base_quadrotor", "lee_velocity_control", "cpu", args=args, num_envs=n)


def _three_substep_env():
    """dynamic_env with exactly 3 physics sub-steps per env step, registered as its own config (the registry hands out the config
    classes themselves, so the shared dynamic_env config must not be changed)"""
    from aerial_gym_simulator_b200.config.env_config import DynamicEnvironmentCfg as dyn
    from aerial_gym_simulator_b200.registry._core import env_config_registry

    class Three(dyn):
        class env(dyn.env):
            num_physics_steps_per_env_step_mean = 3
            num_physics_steps_per_env_step_std = 0
    env_config_registry.register("contact_obstacle_three_substep_test_env", Three)
    return "contact_obstacle_three_substep_test_env"


def _pair_depths(rows, boxes, af, active):
    """the SAT overlap (float64, > 0 when the boxes overlap) of every pair of active assets, per env: {(e, i, j): depth}"""
    out = {}
    P = _params(contact_offset=0.0)
    for e in range(rows.shape[0]):
        idx = np.nonzero(active[e])[0]
        X = {a: CO.box_world(rows[e, a], boxes[af[e, a]]) for a in idx}
        for ii, i in enumerate(idx):
            for j in idx[ii + 1:]:
                if not CO.box_near(P, X[i], X[j]):
                    continue
                c, _ = CO.box_pair(P, X[i], X[j])
                if c:
                    (ci, ai, hi), (cj, aj, hj) = _world_boxes(rows[e, i], boxes[af[e, i]]), _world_boxes(rows[e, j], boxes[af[e, j]])
                    n = np.array(c[0][1], np.float64)
                    out[(e, i, j)] = _support(ci, ai, hi, n) + _support(cj, aj, hj, -n)
    return out


def test_a_dynamic_env_reset_is_pulled_apart_within_the_depenetration_bound():
    """256 envs of dynamic_env after a reset: the overlapping pairs of in-play assets are pushed apart, sub-step after sub-step
    (the advance without twist, then the solve), at up to max_depenetration_velocity each.  A pair d deep needs (d - rest_offset)
    / (v_max dt) sub-steps when nothing else pushes it; piles need a few more, so the bound is twice that plus 10.  At the end no
    pair is deeper than rest_offset + v_max dt: the last solve's target leaves at most one sub-step of travel at the cap."""
    from tests._cpu_stack import cpu_stack
    with cpu_stack() as proxy:
        env = _dynamic_env(256)
        env.reset()
    assert proxy.calls == {}
    P = env.contact_params
    rows = env.global_tensor_dict["env_asset_state_tensor"].numpy().copy()
    mass, boxes, af = env._obstacle_mass.table.numpy(), env._obstacle_boxes.boxes.numpy(), env._obstacle_boxes.asset_file.numpy()
    active = rows[..., 2] > -500.0
    d0 = _pair_depths(rows, boxes, af, active)
    deep = {k: v for k, v in d0.items() if v > P.rest_offset}
    assert len(deep) > 50, len(deep)
    vmax, dt = P.max_depenetration_velocity, P.dt
    bound = int(np.ceil(2 * (max(deep.values()) - P.rest_offset) / (vmax * dt))) + 10
    half = np.float32(0.5)
    for _ in range(bound):
        rows[..., 0:3] += rows[..., 7:10] * np.float32(dt)  # the advance without damping: pose with the current twist
        h, q = rows[..., 10:13] * np.float32(dt) * half, rows[..., 3:7].copy()
        qn = np.stack([q[..., 0] + h[..., 0] * q[..., 3] + h[..., 1] * q[..., 2] - h[..., 2] * q[..., 1],
                       q[..., 1] - h[..., 0] * q[..., 2] + h[..., 1] * q[..., 3] + h[..., 2] * q[..., 0],
                       q[..., 2] + h[..., 0] * q[..., 1] - h[..., 1] * q[..., 0] + h[..., 2] * q[..., 3],
                       q[..., 3] - h[..., 0] * q[..., 0] - h[..., 1] * q[..., 1] - h[..., 2] * q[..., 2]], -1)
        rows[..., 3:7] = qn / np.linalg.norm(qn, axis=-1, keepdims=True)
        obstacle_obstacle_shadow(P, rows, mass, boxes, af)
    d1 = _pair_depths(rows, boxes, af, active)
    worst = max(d1.values(), default=0.0)
    assert worst <= P.rest_offset + vmax * dt, (worst, bound)
    assert all(d1.get(k, 0.0) <= P.rest_offset + vmax * dt for k in deep)


def test_argument_validation(tmp_path):
    from aerial_gym_simulator_b200.config import asset_config as ac
    from aerial_gym_simulator_b200.config.env_config import DynamicEnvironmentCfg as dyn
    from aerial_gym_simulator_b200.env_manager import EnvManager
    from aerial_gym_simulator_b200.hp2 import ContactMotion, ObstacleMass, obstacle_obstacle_contact
    from aerial_gym_simulator_b200.registry._core import env_config_registry
    from tests._cpu_stack import cpu_stack

    base = {"contact": "rigid", "contact_moving_obstacles": True, "contact_dynamic_obstacles": True}
    for bad, what in (({**base, "contact_obstacle_obstacle": 1}, "must be a bool"), ({**base, "contact_obstacle_obstacle": "yes"}, "must be a bool"),
                      ({**base, "contact_dynamic_obstacles": False, "contact_obstacle_obstacle": True}, "needs args\\['contact_dynamic_obstacles'\\]"),
                      ({"contact": "rigid", "contact_obstacle_obstacle": True}, "needs args\\['contact_dynamic_obstacles'\\]")):
        with pytest.raises(ValueError, match="contact_obstacle_obstacle.*" + what):
            EnvManager("base_sim", "dynamic_env", "base_quadrotor", "lee_velocity_control", "cpu", args=bad, num_envs=2)
    # an asset that is not exactly one box, named in the error
    body = '<inertial><mass value="1.0"/><inertia ixx="1" ixy="0" ixz="0" iyy="1" iyz="0" izz="1"/></inertial>'
    for name, geo in (("cyl.urdf", '<visual><geometry><cylinder radius="0.1" length="1.0"/></geometry></visual>'),
                      ("two_boxes.urdf", '<visual><geometry><box size="0.1 0.1 0.1"/></geometry></visual>'
                                         '<visual><origin xyz="0.3 0 0"/><geometry><box size="0.1 0.1 0.1"/></geometry></visual>')):
        d = tmp_path / name.split(".")[0]
        d.mkdir()
        (d / name).write_text(f'<?xml version="1.0"?><robot name="x"><link name="base_link">{body}{geo}</link></robot>')

        class Obj(ac.dynamic_object_asset_params):
            asset_folder = str(d)
            num_assets = 3

        class Env(dyn):
            class env_config(dyn.env_config):
                asset_type_to_dict_map = {**dyn.env_config.asset_type_to_dict_map, "objects": Obj}
        env_config_registry.register(f"contact_obstacle_{name}_test_env", Env)
        with cpu_stack():
            with pytest.raises(ValueError, match=f"{name}.*exactly one <box>"):
                EnvManager("base_sim", f"contact_obstacle_{name}_test_env", "base_quadrotor", "lee_velocity_control", "cpu",
                           args={**base, "contact_obstacle_obstacle": True}, num_envs=2)
            EnvManager("base_sim", f"contact_obstacle_{name}_test_env", "base_quadrotor", "lee_velocity_control", "cpu", args=base,
                       num_envs=2)
    # the box table
    E, A = 3, 4
    bx = torch.from_numpy(_boxes())
    af = torch.zeros(E, A, dtype=torch.int64)
    t = ObstacleBoxes(bx, af)
    assert (t.E, t.A, t.F) == (E, A, 5) and t.asset_file.dtype == torch.int32
    nan, neg, skew = bx.clone(), bx.clone(), bx.clone()
    nan[1, 4] = float("nan")
    neg[2, 13] = -0.1
    skew[0, 3:6] = torch.tensor([1.0, 0.1, 0.0])
    for args in ((bx.int(), af), (bx, af.float()), (bx[:, :14], af), (bx[:0], af), (bx, af[0]), (nan, af), (neg, af), (skew, af),
                 (bx, af + 5), (bx, af - 1)):
        with pytest.raises(ValueError):
            ObstacleBoxes(*args)
    # the launch wrapper
    st = torch.zeros(E, A, 13)
    mo, ms = ContactMotion(st, torch.zeros(E, 2, dtype=torch.int32)), ObstacleMass(torch.zeros(E, A, 13))
    p = _params()
    for args in ((p, st, ms, t), (None, mo, ms, t), (p, mo, ms.table, t), (p, mo, ms, None),
                 (p, mo, ObstacleMass(torch.zeros(E, A + 1, 13)), t), (p, mo, ms, ObstacleBoxes(bx, af[:2]))):
        with pytest.raises(ValueError):
            obstacle_obstacle_contact(*args)
    big = torch.zeros(E, 65, 13)
    with pytest.raises(ValueError, match="at most 64"):
        obstacle_obstacle_contact(p, ContactMotion(big, torch.zeros(E, 1, dtype=torch.int32)), ObstacleMass(torch.zeros(E, 65, 13)),
                                  ObstacleBoxes(bx, torch.zeros(E, 65, dtype=torch.int32)))
    with pytest.raises(_lib.AgxError, match="CUDA"):
        obstacle_obstacle_contact(p, mo, ms, t)
    # the C entry point, NULL tables included
    lib = _lib.load()
    assert lib.agx_sizeof(16) == C.sizeof(_lib.AgxObstacleBoxes) == 24
    pm = C.c_void_p(ms.table.data_ptr())
    f = lib.agx_obstacle_obstacle_contact
    assert f(E, A, C.byref(p), None, 13, pm, None, None) == -3
    assert f(E, A, C.byref(p), None, 13, None, C.byref(t.c), None) == -3
    assert f(E, A, None, None, 13, pm, C.byref(t.c), None) == -3
    assert f(E, A, C.byref(p), None, 12, pm, C.byref(t.c), None) == -1
    assert f(-1, A, C.byref(p), None, 13, pm, C.byref(t.c), None) == -1
    assert f(E, 65, C.byref(p), None, 13, pm, C.byref(t.c), None) == -1
    assert f(E, A, C.byref(p), None, 13, pm, C.byref(t.c), None) == -3  # asset_state NULL
    assert f(0, A, C.byref(p), None, 13, pm, C.byref(t.c), None) == 0 and f(E, 1, C.byref(p), None, 13, pm, C.byref(t.c), None) == 0
    for bad in (_lib.AgxObstacleBoxes(boxes=None, asset_file=t.c.asset_file, num_files=5),
                _lib.AgxObstacleBoxes(boxes=t.c.boxes, asset_file=None, num_files=5)):
        assert f(E, A, C.byref(p), None, 13, pm, C.byref(bad), None) == -3
    assert f(E, A, C.byref(p), None, 13, pm, C.byref(_lib.AgxObstacleBoxes(boxes=t.c.boxes, asset_file=t.c.asset_file, num_files=0)),
             None) == -1
    assert f(E, A, C.byref(_params(dt=0.0)), None, 13, pm, C.byref(t.c), None) == -1


def test_dynamic_env_end_to_end_on_the_cpu_stack():
    """dynamic_env with every contact key on the CPU twins: each sub-step runs the obstacle advance, the ground solve, the
    obstacle-obstacle solve, the re-pose and the robot's solve in that order, and the obstacle rows after an env step equal a
    replay of that order with the shadows"""
    from tests._cpu_stack import cpu_stack
    with cpu_stack() as proxy, obstacle_twins() as log:
        env = _dynamic_env(16, seed=3, env_name=_three_substep_env(), contact_obstacle_ground=True, step_mode="launch")
        env.reset()
        ast = env.global_tensor_dict["env_asset_state_tensor"]
        before = ast.numpy().copy()
        log.clear()
        g = torch.Generator().manual_seed(4)
        tw = (torch.rand(16, env.num_obs_in_env, 6, generator=g) * 2 - 1) * 0.5
        env.step(actions=torch.zeros(16, env.num_robot_actions), env_actions=tw)
        after = ast.numpy().copy()
        env.step(actions=torch.zeros(16, env.num_robot_actions))  # a step without env_actions drifts with the solved twists
    assert proxy.calls == {}  # every sub-step ran on the twins: no library entry point was reached
    seq = [x for x in log if x != "repose"]
    assert seq[:9] == ["obstacle_ground", "obstacle_obstacle", "robot_contact"] * 3
    assert not np.array_equal(before, after)
    # replay: the advance (the shadow of agx_obstacle_step), the ground shadow, the pair shadow, three times
    from tests import _shadow
    P, mass, boxes, af = env.contact_params, env._obstacle_mass.table.numpy(), env._obstacle_boxes.boxes.numpy(), env._obstacle_boxes.asset_file.numpy()
    hull = env._obstacle_hull
    rows = before.copy()
    E, A = rows.shape[:2]
    t = np.ascontiguousarray(tw.numpy(), np.float32)
    for _ in range(3):
        _shadow.load().shadow_obstacle_step(E, A, C.c_void_p(rows.ctypes.data), 13, C.c_void_p(t.ctypes.data),
                                            env.sim_config.sim.dt, 1, env._asset_damping[0], env._asset_damping[1])
        ground_shadow(P, rows, mass, hull)
        obstacle_obstacle_shadow(P, rows, mass, boxes, af)
    assert np.array_equal(rows, after)
