"""Obstacle-ground contact on the CPU: contact_core.cuh's obstacle_ground_row (compiled for the host) against
oracle/contact_ground_oracle.py bit for bit, untouched rows, the kept vertex set, a box driven into the ground, the depenetration
cap, energy that never rises, the Coulomb bound, a corner landing, and the argument checks."""
import ctypes as C

import numpy as np
import pytest
import torch

from aerial_gym_simulator_b200 import _lib
from aerial_gym_simulator_b200.env_manager.env_manager import _hull_vertices
from aerial_gym_simulator_b200.hp2 import ObstacleHull, box_triangles, cylinder_triangles, icosphere_triangles
from oracle import contact_dynamic_oracle as CD
from oracle import contact_ground_oracle as CG
from tests import _contact_ground_shadow
from tests.test_contact_cpu import params

_p = lambda a: C.c_void_p(a.ctypes.data)
CMAX = CG.CONTACT_MAX


def _rot(axis, ang):
    a = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(ang) * K + (1 - np.cos(ang)) * K @ K


def _part(tris, R=np.eye(3), p=(0.0, 0.0, 0.0)):
    t = np.asarray(tris, np.float64).reshape(-1, 3)
    return ("link", 0, (t @ R.T + np.asarray(p)).reshape(-1, 9).astype(np.float32), None)


def _tree():
    """a trunk and three branches of tessellated cylinders, as the trees' URDFs are built"""
    parts = [_part(cylinder_triangles(0.12, 3.0), p=(0.0, 0.0, 1.5))]
    for k, (h, yaw) in enumerate([(1.2, 0.3), (1.9, 2.4), (2.5, 4.4)]):
        R = _rot((np.cos(yaw), np.sin(yaw), 0.0), 0.9 + 0.2 * k) @ _rot((0, 0, 1), yaw)
        parts.append(_part(cylinder_triangles(0.05, 1.0), R, np.array([0.0, 0.0, h]) + R @ np.array([0.0, 0.0, 0.5])))
    return parts


def _files():
    """per-file vertex arrays: two boxes, a tree-like multi-cylinder asset, an icosphere"""
    return [_hull_vertices([_part(box_triangles((0.4, 0.3, 0.2)))]), _hull_vertices([_part(box_triangles((2.0, 0.1, 0.1)))]),
            _hull_vertices(_tree()), _hull_vertices([_part(icosphere_triangles(0.3))])]


def _hull(files, asset_file):
    h = ObstacleHull.from_files(files, np.asarray(asset_file).reshape(-1, 1), "cpu")  # rows as [R,1]
    return h.vertices.numpy(), h.file_offset.numpy(), h.file_reach.numpy(), h.asset_file.numpy().reshape(-1)


def _box_mass(m, size):
    J = np.diag([size[1] ** 2 + size[2] ** 2, size[0] ** 2 + size[2] ** 2, size[0] ** 2 + size[1] ** 2]) * m / 12.0
    return np.concatenate([[1.0 / m], [0.0, 0.0, 0.0], np.linalg.inv(J).reshape(9)]).astype(np.float32)


def random_rows(R, nfiles, seed, kinematic=0.15, vscale=3.0):
    """rows straddling the plane (z in [-1, 2.5]), random orientations, |v| <= vscale, |w| <= 2; a mass table with a `kinematic`
    fraction of all-zero rows, the others 0.1-13 kg with a COM up to 1.5 m off the origin and a full symmetric inverse inertia"""
    g = np.random.default_rng(seed)
    rows = np.zeros((R, 13), np.float32)
    rows[:, 0:2] = g.uniform(-3, 3, (R, 2))
    rows[:, 2] = g.uniform(-1.0, 2.5, R)
    q = g.normal(size=(R, 4))
    rows[:, 3:7] = q / np.linalg.norm(q, axis=1, keepdims=True)
    d = g.normal(size=(R, 6))
    rows[:, 7:10] = d[:, 0:3] / np.linalg.norm(d[:, 0:3], axis=1, keepdims=True) * g.uniform(0, vscale, (R, 1))
    rows[:, 10:13] = d[:, 3:6] / np.linalg.norm(d[:, 3:6], axis=1, keepdims=True) * g.uniform(0, 2, (R, 1))
    mass = np.zeros((R, 13), np.float32)
    m = np.exp(g.uniform(np.log(0.1), np.log(13.0), R))
    mass[:, 0] = 1.0 / m
    mass[:, 1:4] = g.uniform(-1, 1, (R, 3)) * g.choice([0.0, 0.2, 1.5], (R, 1))
    M = g.normal(size=(R, 3, 3))
    J = (M @ np.swapaxes(M, -1, -2) + np.eye(3)) * m[:, None, None] * 0.2
    mass[:, 4:13] = np.linalg.inv(J).reshape(R, 9)
    mass[g.uniform(size=R) < kinematic] = 0.0
    return rows, mass, g.integers(0, nfiles, R).astype(np.int32)


def shadow_ground(p, rows, mass, verts, off, reach, af):
    st = np.ascontiguousarray(rows, np.float32).copy()
    R = st.shape[0]
    kept = np.zeros((R, CMAX), np.int32)
    count = np.zeros(R, np.int32)
    _contact_ground_shadow.load().shadow_obstacle_ground(
        R, C.byref(p), _p(st), st.shape[1], _p(np.ascontiguousarray(mass, np.float32)), _p(np.ascontiguousarray(verts, np.float32)),
        _p(np.ascontiguousarray(off, np.int32)), _p(np.ascontiguousarray(reach, np.float32)), _p(np.ascontiguousarray(af, np.int32)),
        _p(kept), _p(count))
    return st, kept, count


def _ground_params(**kw):
    d = dict(contact_offset=0.002, rest_offset=0.001, dt=0.01, friction=1.0, max_depenetration_velocity=1.0, iterations=4)
    d.update(kw)
    return params(**d)


@pytest.mark.parametrize("iterations,friction,seed", [(1, 0.0, 0), (4, 1.0, 1), (10, 0.5, 2), (4, 2.0, 3)])
def test_shadow_matches_oracle_bit_for_bit(iterations, friction, seed):
    files = _files()
    rows, mass, af = random_rows(3000, len(files), seed)
    verts, off, reach, af = _hull(files, af)
    p = _ground_params(iterations=iterations, friction=friction)
    got, kept, count = shadow_ground(p, rows, mass, verts, off, reach, af)
    ref, ref_kept, ref_count = CG.ground_contact(p, rows, mass, verts, off, reach, af)
    assert np.array_equal(count, ref_count) and np.array_equal(kept, ref_kept), f"{(kept != ref_kept).any(1).sum()} kept sets differ"
    assert np.array_equal(got, ref), f"{(got != ref).any(1).sum()} rows differ"
    # every file and every count occurs; only rows with a kept contact change (a separating one may keep its values)
    touched = count > 0
    assert set(af[touched]) == set(range(len(files))) and (count == CMAX).any() and ((count > 0) & (count < CMAX)).any()
    changed = (got != rows).any(axis=1)
    assert not changed[~touched].any() and changed[touched].mean() > 0.5
    assert 0.2 < touched.mean() < 0.8


def test_rows_clear_of_the_ground_and_kinematic_rows_are_untouched():
    files = _files()
    rows, mass, af = random_rows(2000, len(files), 4, kinematic=0.5)
    verts, off, reach, af = _hull(files, af)
    p = _ground_params()
    low = CG.lowest_vertex(rows, verts, off, af)
    got, kept, count = shadow_ground(p, rows, mass, verts, off, reach, af)
    clear = low > p.contact_offset + 1e-6
    kinematic = ~mass.any(axis=1)
    assert clear.sum() > 300 and (kinematic & (low < -0.1)).sum() > 100
    for m in (clear, kinematic):
        assert np.array_equal(got[m], rows[m]) and not count[m].any() and (kept[m] == -1).all()
    assert count[~clear & ~kinematic].min() > 0


def _one(p, row, mass, verts):
    verts = np.asarray(verts, np.float32).reshape(-1, 3)
    vt, off, reach, af = _hull([verts], np.zeros((1, 1), np.int32))
    got, kept, count = shadow_ground(p, np.asarray(row, np.float32)[None], np.asarray(mass, np.float32)[None], vt, off, reach, af)
    ref, ref_kept, _ = CG.ground_contact(p, np.asarray(row, np.float32)[None], np.asarray(mass, np.float32)[None], vt, off, reach, af)
    assert np.array_equal(got, ref) and np.array_equal(kept, ref_kept)
    return got[0], kept[0, :count[0]]


def _row(x, q=(0.0, 0.0, 0.0, 1.0), v=(0.0, 0.0, 0.0), w=(0.0, 0.0, 0.0)):
    return np.concatenate([x, q, v, w]).astype(np.float32)


def test_selection_keeps_the_deepest_with_ties_to_the_lower_index():
    p = _ground_params()
    box = _hull_vertices([_part(box_triangles((0.4, 0.3, 0.2)))])
    assert len(box) == 8
    _, kept = _one(p, _row((0.0, 0.0, 0.1 - 0.0005)), _box_mass(1.0, (0.4, 0.3, 0.2)), box)
    assert sorted(kept) == sorted(np.nonzero(box[:, 2] < 0)[0]) and len(kept) == 4  # a flat box: its 4 bottom vertices
    # 12 vertices on one level and 3 deeper ones: the 3 deepest (deepest first), then the 5 lowest indices of the level
    g = np.random.default_rng(5)
    v = np.zeros((15, 3), np.float32)
    v[:, 0:2] = g.uniform(-1, 1, (15, 2))
    deep = [13, 4, 9]
    v[deep, 2] = [-0.3, -0.2, -0.1]
    _, kept = _one(p, _row((0.0, 0.0, 0.0)), _box_mass(1.0, (1.0, 1.0, 1.0)), v)
    level = [i for i in range(15) if i not in deep]
    assert list(kept) == deep + level[:5]
    # a vertex exactly at contact_offset is not a candidate, one just below is
    v2 = np.array([[0.0, 0.0, 0.0], [0.5, 0.0, 0.0]], np.float32)
    z = np.float32(p.contact_offset)
    row = _row((0.0, 0.0, z))
    row[2] = z
    _, kept = _one(p, row, _box_mass(1.0, (1.0, 1.0, 1.0)), v2)
    assert len(kept) == 0
    row[2] = np.nextafter(z, np.float32(-1))
    _, kept = _one(p, row, _box_mass(1.0, (1.0, 1.0, 1.0)), v2)
    assert list(kept) == [0, 1]


def _drive(p, row, mass, verts, steps, twist=None):
    """per sub-step: the twist rewritten (if given), x += v dt and q advanced as agx_obstacle_step does without damping, then one
    ground-contact launch; returns the rows after each sub-step"""
    vt, off, reach, af = _hull([verts], np.zeros((1, 1), np.int32))
    r, out = np.asarray(row, np.float32)[None].copy(), []
    dt, half = np.float32(p.dt), np.float32(0.5)
    for _ in range(steps):
        if twist is not None:
            r[0, 7:13] = twist
        r[0, 0:3] = r[0, 0:3] + r[0, 7:10] * dt
        h, q = r[0, 10:13] * dt * half, r[0, 3:7].copy()
        qn = np.array([q[0] + h[0] * q[3] + h[1] * q[2] - h[2] * q[1], q[1] - h[0] * q[2] + h[1] * q[3] + h[2] * q[0],
                       q[2] + h[0] * q[1] - h[1] * q[0] + h[2] * q[3], q[3] - h[0] * q[0] - h[1] * q[1] - h[2] * q[2]], np.float32)
        r[0, 3:7] = qn / np.sqrt((qn * qn).sum())
        r, _, _ = shadow_ground(p, r, np.asarray(mass, np.float32)[None], vt, off, reach, af)
        out.append(r[0].copy())
    return np.asarray(out), vt, off, af


def test_a_box_driven_down_at_2_m_s_stops_at_the_ground():
    p = _ground_params()
    size = (0.4, 0.3, 0.2)
    box = _hull_vertices([_part(box_triangles(size))])
    twist = np.array([0.3, -0.2, -2.0, 0.0, 0.0, 0.0], np.float32)
    hist, vt, off, af = _drive(p, _row((0.0, 0.0, 0.5)), _box_mass(1.0, size), box, 150, twist)
    depth = -CG.lowest_vertex(hist, vt, off, np.zeros(len(hist), np.int32))
    # after each sub-step (advance, then solve) the lowest vertex is at most rest_offset + one sub-step of travel deep; once landed
    # it stays within that band: the solve's position correction leaves it about one sub-step of travel above the plane, and the
    # next advance brings it back to the rest offset, so it neither sinks nor leaves
    band = p.rest_offset + 2.0 * p.dt
    assert depth.max() <= band + 1e-5, depth.max()
    landed = np.nonzero(depth > -(band + p.contact_offset))[0][0]
    assert landed < 30 and depth[landed:].min() > -(band + p.contact_offset) and depth[landed:].max() <= p.rest_offset + 1e-5
    assert hist[-1, 9] >= -1e-5  # the commanded -2 m/s is cancelled at the ground every sub-step


@pytest.mark.parametrize("under", [0.5, 1000.0])
def test_an_obstacle_under_the_ground_rises_at_the_depenetration_cap(under):
    p = _ground_params(iterations=10)
    size = (0.4, 0.3, 0.2)
    box = _hull_vertices([_part(box_triangles(size))])
    row, kept = _one(p, _row((0.2, -0.1, -under)), _box_mass(1.0, size), box)
    assert len(kept) == 8
    maxd = np.float32(p.max_depenetration_velocity)
    assert abs(row[9] - maxd) <= 1e-6 * maxd and np.abs(row[[7, 8, 10, 11, 12]]).max() <= 1e-6, row[7:13]
    assert abs((row[2] - np.float32(-under)) - p.dt * maxd) <= 1e-6 * max(under, 1.0)
    # and again the next sub-step: not faster
    hist, *_ = _drive(p, row, _box_mass(1.0, size), box, 5)
    assert np.abs(hist[:, 9] - maxd).max() <= 1e-6 * maxd


def test_kinetic_energy_never_rises_without_bias():
    files = _files()
    rows, mass, af = random_rows(2000, len(files), 6, kinematic=0.0)
    verts, off, reach, af = _hull(files, af)
    for friction in (0.0, 0.5, 2.0):
        p = _ground_params(friction=friction, rest_offset=0.004, contact_offset=0.006)
        low = CG.lowest_vertex(rows, verts, off, af)
        r = rows.copy()
        r[:, 2] += (np.random.default_rng(7).uniform(-0.004, 0.006, len(r)) - low).astype(np.float32)  # depth <= rest_offset
        lowr = CG.lowest_vertex(r, verts, off, af)
        assert lowr.min() >= -0.004 - 1e-5
        got, _, count = shadow_ground(p, r, mass, verts, off, reach, af)
        checked = 0
        for i in np.nonzero(count)[0]:
            m, com, J = 1.0 / float(mass[i, 0]), mass[i, 1:4], np.linalg.inv(mass[i, 4:13].astype(np.float64).reshape(3, 3))
            after = r[i].copy()
            after[7:13] = got[i, 7:13]  # the solve's twist on the pose it ran with
            e0, e1 = CD.body_energy(r[i], m, com, J), CD.body_energy(after, m, com, J)
            assert e1 <= e0 * (1 + 1e-5) + 1e-7, (friction, i, e0, e1)
            checked += 1
        assert checked > 1000


def _com_velocity(row, mass):
    R = CD._R64(row[3:7])
    c = row[0:3].astype(np.float64) + R @ mass[1:4].astype(np.float64)
    return row[7:10].astype(np.float64) + np.cross(row[10:13].astype(np.float64), c - row[0:3])


@pytest.mark.parametrize("mu", [0.2, 0.5, 1.0])
def test_an_oblique_impact_obeys_coulomb(mu):
    p = _ground_params(friction=mu, iterations=10)
    size = (0.4, 0.4, 0.4)
    box = _hull_vertices([_part(box_triangles(size))])
    g = np.random.default_rng(8)
    for _ in range(20):
        q = g.normal(size=4)
        q /= np.linalg.norm(q)
        row = _row((0.0, 0.0, 0.0), q, (g.uniform(-4, 4), g.uniform(-4, 4), -g.uniform(0.5, 3)), g.normal(size=3) * 0.5)
        vt, off, _, af = _hull([box], np.zeros((1, 1), np.int32))
        row[2] = -CG.lowest_vertex(row[None], vt, off, af)[0] - 0.0005  # lowest vertex 0.5 mm deep: below rest_offset, no bias
        m = _box_mass(1.0, size)
        after, kept = _one(p, row, m, box)
        assert len(kept) >= 1
        dv = _com_velocity(after, m) - _com_velocity(row, m)
        assert dv[2] > 0 and np.linalg.norm(dv[0:2]) <= mu * dv[2] * (1 + 1e-5) + 1e-6, (dv, mu)


def test_a_corner_landing_spins_the_box_by_its_lever_arm():
    p = _ground_params(friction=0.0)
    size = (0.4, 0.4, 0.4)
    box = _hull_vertices([_part(box_triangles(size))])
    m = _box_mass(1.0, size)
    for axis, ang in (((1.0, 0.7, 0.0), 0.5), ((-0.4, 1.0, 0.2), 0.7), ((0.3, -1.0, 0.5), 0.9)):
        Rm = _rot(axis, ang)
        w_, x_, y_, z_ = np.cos(ang / 2), *(np.sin(ang / 2) * np.asarray(axis) / np.linalg.norm(axis))
        q = np.array([x_, y_, z_, w_])
        world = box.astype(np.float64) @ Rm.T
        low = int(np.argmin(world[:, 2]))
        assert np.sort(world[:, 2])[1] - world[low, 2] > 0.02  # one corner clearly lowest
        row = _row((0.0, 0.0, -world[low, 2] - 0.0005), q, (0.0, 0.0, -2.0))
        after, kept = _one(p, row, m, box)
        assert list(kept) == [low]
        r = world[low]  # lever arm from the COM (the origin) to the corner
        w = after[10:13]
        # impulse +z at r: dw ~ r x z = (r_y, -r_x, 0) for the cube's isotropic inertia
        assert np.sign(w[0]) == np.sign(r[1]) and np.sign(w[1]) == -np.sign(r[0]) and abs(w[2]) < 1e-5, (w, r)
        assert after[9] > -2.0  # and the fall slows


def test_argument_validation():
    from aerial_gym_simulator_b200.env_manager import EnvManager
    from aerial_gym_simulator_b200.hp2 import ContactMotion, ObstacleMass, obstacle_ground_contact

    base = {"contact": "rigid", "contact_moving_obstacles": True, "contact_dynamic_obstacles": True}
    for bad, what in (({**base, "contact_obstacle_ground": 1}, "bool"), ({**base, "contact_obstacle_ground": "yes"}, "bool"),
                      ({**base, "contact_dynamic_obstacles": False, "contact_obstacle_ground": True}, "contact_dynamic_obstacles"),
                      ({"contact": "rigid", "contact_obstacle_ground": True}, "contact_dynamic_obstacles")):
        with pytest.raises(ValueError, match="contact_obstacle_ground"):
            EnvManager("base_sim", "dynamic_env", "base_quadrotor", "lee_velocity_control", "cpu", args=bad, num_envs=2)
    from aerial_gym_simulator_b200.config.env_config import DynamicEnvironmentCfg as dyn
    from aerial_gym_simulator_b200.registry._core import env_config_registry

    class NoGround(dyn):
        class env(dyn.env):
            create_ground_plane = False
    env_config_registry.register("contact_ground_no_plane_test_env", NoGround)
    with pytest.raises(ValueError, match="create_ground_plane"):
        EnvManager("base_sim", "contact_ground_no_plane_test_env", "base_quadrotor", "lee_velocity_control", "cpu",
                   args={**base, "contact_obstacle_ground": True}, num_envs=2)
    # the hull table
    E, A = 3, 4
    v = torch.tensor(_hull_vertices([_part(box_triangles((1.0, 1.0, 1.0)))]))
    off, reach, af = torch.tensor([0, 8]), torch.tensor([0.87]), torch.zeros(E, A, dtype=torch.int64)
    h = ObstacleHull(v, off, reach, af)
    assert (h.E, h.A, h.F) == (E, A, 1) and h.asset_file.dtype == torch.int32 and h.file_offset.dtype == torch.int32
    nan = v.clone()
    nan[3, 1] = float("nan")
    for args in ((v.double().int(), off, reach, af), (v, off.float(), reach, af), (v, off, reach, af.float()),
                 (v[:, :2], off, reach, af), (v, torch.tensor([0, 4, 8]), reach, af), (v, off, torch.zeros(0), af),
                 (v, off, reach, af[0]), (nan, off, reach, af), (v, off, torch.tensor([float("inf")]), af),
                 (v, off, torch.tensor([-1.0]), af), (v, torch.tensor([1, 8]), reach, af), (v, torch.tensor([0, 7]), reach, af),
                 (v, torch.tensor([0, 9, 8]), torch.tensor([1.0, 1.0]), af), (v, off, reach, af + 1), (v, off, reach, af - 1)):
        with pytest.raises(ValueError):
            ObstacleHull(*args)
    hf = ObstacleHull.from_files([np.asarray(v), np.zeros((0, 3), np.float32), np.asarray(v) * 2], np.array([[0, 2], [1, 2]]), "cpu")
    assert hf.file_offset.tolist() == [0, 8, 8, 16] and hf.file_reach[0] > np.sqrt(0.75) and hf.file_reach[2] > np.sqrt(3.0)
    assert float(hf.file_reach[0]) == float(np.nextafter(np.float32(np.sqrt(0.75)), np.float32(np.inf)))
    # the launch wrapper
    st = torch.zeros(E, A, 13)
    mo, ms = ContactMotion(st, torch.zeros(E, 2, dtype=torch.int32)), ObstacleMass(torch.zeros(E, A, 13))
    p = _ground_params()
    for args in ((p, st, ms, h), (None, mo, ms, h), (p, mo, ms.table, h), (p, mo, ms, None),
                 (p, mo, ObstacleMass(torch.zeros(E, A + 1, 13)), h), (p, mo, ms, ObstacleHull(v, off, reach, af[:2]))):
        with pytest.raises(ValueError):
            obstacle_ground_contact(*args)
    with pytest.raises(_lib.AgxError, match="CUDA"):
        obstacle_ground_contact(p, mo, ms, h)
    # the C entry point
    lib = _lib.load()
    assert lib.agx_sizeof(14) == C.sizeof(_lib.AgxObstacleHull) == 40
    pm = C.c_void_p(ms.table.data_ptr())
    assert lib.agx_obstacle_ground_contact(E, A, C.byref(p), None, 13, pm, None, None) == -3
    assert lib.agx_obstacle_ground_contact(E, A, C.byref(p), None, 13, None, C.byref(h.c), None) == -3
    assert lib.agx_obstacle_ground_contact(E, A, None, None, 13, pm, C.byref(h.c), None) == -3
    assert lib.agx_obstacle_ground_contact(E, A, C.byref(p), None, 12, pm, C.byref(h.c), None) == -1
    assert lib.agx_obstacle_ground_contact(-1, A, C.byref(p), None, 13, pm, C.byref(h.c), None) == -1
    assert lib.agx_obstacle_ground_contact(E, A, C.byref(p), None, 13, pm, C.byref(h.c), None) == -3  # asset_state NULL
    assert lib.agx_obstacle_ground_contact(0, A, C.byref(p), None, 13, pm, C.byref(h.c), None) == 0  # nothing to do
    bad = _lib.AgxObstacleHull(vertices=h.c.vertices, file_offset=None, file_reach=h.c.file_reach, asset_file=h.c.asset_file, num_files=1)
    assert lib.agx_obstacle_ground_contact(E, A, C.byref(p), None, 13, pm, C.byref(bad), None) == -3
    bad.file_offset, bad.num_files = h.c.file_offset, 0
    assert lib.agx_obstacle_ground_contact(E, A, C.byref(p), None, 13, pm, C.byref(bad), None) == -1
    p0 = _ground_params(dt=0.0)
    assert lib.agx_obstacle_ground_contact(E, A, C.byref(p0), None, 13, pm, C.byref(h.c), None) == -1
