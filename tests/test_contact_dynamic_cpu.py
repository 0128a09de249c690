"""Rigid contact with dynamic obstacles on the CPU: the two-body solve of contact_core.cuh (compiled for the host) against
oracle/contact_dynamic_oracle.py bit for bit, its reduction to the moving solve at infinite obstacle mass, conservation of momentum,
a head-on collision ending at the common velocity, energy that never rises, multi-part assets as one body, the spin of an
off-centre hit, and the argument checks."""
import ctypes as C

import numpy as np
import pytest
import torch

from aerial_gym_simulator_b200 import _lib
from oracle import contact_dynamic_oracle as CD
from oracle import contact_moving_oracle as CM
from oracle import contact_oracle as CO
from tests import _contact_dynamic_shadow
from tests.test_contact_cpu import params, random_contact_sets
from tests.test_contact_moving_cpu import _full_params, shadow_moving

_p = lambda a: C.c_void_p(a.ctypes.data)
CMAX = CO.CONTACT_MAX
K_OBJ, A_AST = 9, 5  # objects and assets per env of the random sets


def random_bodies(root, cts, count, seed, kinematic=0.2, ground=True):
    """ids (distinct objects, the ground K_OBJ at most once), obj_asset [E,K_OBJ] -> [0,A_AST), asset rows within 1 m of the robot with
    |v| <= 3 m/s and |w| <= 2 rad/s, and a mass table: a `kinematic` fraction of all-zero rows, the others 0.1-10 kg with a COM up
    to 3 m off the origin and a full symmetric inverse inertia"""
    E = root.shape[0]
    g = np.random.default_rng(seed)
    count = np.minimum(count, K_OBJ + (1 if ground else 0))
    ids = np.full((E, CMAX), -1, np.int32)
    for e in range(E):
        ids[e, :count[e]] = g.permutation(K_OBJ + (1 if ground else 0))[:count[e]]
    obj_asset = g.integers(0, A_AST, (E, K_OBJ)).astype(np.int32)
    rows = np.zeros((E, A_AST, 13), np.float32)
    rows[..., 0:3] = root[:, None, 0:3] + g.uniform(-1, 1, (E, A_AST, 3))
    q = g.normal(size=(E, A_AST, 4))
    rows[..., 3:7] = q / np.linalg.norm(q, axis=-1, keepdims=True)
    d = g.normal(size=(E, A_AST, 6))
    rows[..., 7:10] = d[..., 0:3] / np.linalg.norm(d[..., 0:3], axis=-1, keepdims=True) * g.uniform(0, 3, (E, A_AST, 1))
    rows[..., 10:13] = d[..., 3:6] / np.linalg.norm(d[..., 3:6], axis=-1, keepdims=True) * g.uniform(0, 2, (E, A_AST, 1))
    mass = np.zeros((E, A_AST, 13), np.float32)
    m = np.exp(g.uniform(np.log(0.1), np.log(10.0), (E, A_AST)))
    mass[..., 0] = 1.0 / m
    mass[..., 1:4] = g.uniform(-1, 1, (E, A_AST, 3)) * g.choice([0.0, 0.3, 3.0], (E, A_AST, 1))
    M = g.normal(size=(E, A_AST, 3, 3))
    J = (M @ np.swapaxes(M, -1, -2) + np.eye(3)) * m[..., None, None] * 0.2
    mass[..., 4:13] = np.linalg.inv(J).reshape(E, A_AST, 9)
    mass[g.uniform(size=(E, A_AST)) < kinematic] = 0.0
    return count.astype(np.int32), ids, obj_asset, rows, mass


def shadow_dynamic(p, root, cts, count, ids, rows, obj_asset, mass):
    got, st = root.copy(), np.ascontiguousarray(rows, np.float32).copy()
    force = np.zeros((root.shape[0], 3), np.float32)
    crash = np.zeros(root.shape[0], np.uint8)
    _contact_dynamic_shadow.load().shadow_contact_solve_dynamic(
        root.shape[0], C.byref(p), _p(got), 13, _p(cts), _p(count), _p(np.ascontiguousarray(ids, np.int32)), obj_asset.shape[1], _p(st),
        st.shape[1], 13, _p(np.ascontiguousarray(obj_asset, np.int32)), _p(np.ascontiguousarray(mass, np.float32)), _p(force), _p(crash))
    return got, force, crash.astype(bool), st


@pytest.mark.parametrize("iterations,friction,seed", [(1, 0.0, 0), (4, 1.0, 1), (10, 0.5, 2), (4, 2.0, 3)])
def test_shadow_dynamic_solve_matches_oracle_bit_for_bit(iterations, friction, seed):
    E = 500
    root, cts, count = random_contact_sets(E, seed)
    count, ids, obj_asset, rows, mass = random_bodies(root, cts, count, seed + 50)
    p = _full_params(iterations=iterations, friction=friction)
    got, force, crash, st = shadow_dynamic(p, root, cts, count, ids, rows, obj_asset, mass)
    ref, ref_f, ref_c, ref_st = CD.solve(p, root, cts, count, ids, rows, obj_asset, mass)
    assert np.array_equal(got, ref), f"{(got != ref).sum()} robot values differ"
    assert np.array_equal(force, ref_f) and np.array_equal(crash, ref_c)
    assert np.array_equal(st, ref_st), f"{(st != ref_st).sum()} asset values differ"
    # free touched assets were written, kinematic and untouched ones not
    body, assets, nb = CD.gather_bodies(ids, count, obj_asset)
    touched = np.zeros((E, A_AST), bool)
    for e in range(E):
        touched[e, assets[e, :nb[e]]] = True
    free = (mass[..., 0] > 0) | (mass[..., 4:] != 0).any(-1)
    assert np.array_equal(st[~(touched & free)], rows[~(touched & free)])
    assert (st[touched & free] != rows[touched & free]).any(axis=1).mean() > 0.5  # the rest separate: no impulse
    # the bodies do change the robot's outcome
    u = CM.obstacle_point_velocity(rows, obj_asset, cts, ids)
    moving, _, _ = CM.solve(p, root, cts, count, obstacle_velocity=u)
    assert not np.array_equal(ref[:, 7:13], moving[:, 7:13])


def test_infinite_mass_is_the_moving_solve_bit_for_bit():
    E = 500
    root, cts, count = random_contact_sets(E, 7)
    count, ids, obj_asset, rows, mass = random_bodies(root, cts, count, 57, kinematic=1.0)
    assert not mass.any()
    p = _full_params(iterations=4, friction=1.0)
    got, force, crash, st = shadow_dynamic(p, root, cts, count, ids, rows, obj_asset, mass)
    u = CM.obstacle_point_velocity(rows, obj_asset, cts, ids)
    mg, mf, mc = shadow_moving(p, root, cts, count, u)
    assert np.array_equal(got, mg) and np.array_equal(force, mf) and np.array_equal(crash, mc)
    assert np.array_equal(st, rows)  # rows untouched
    ref, ref_f, _, ref_st = CD.solve(p, root, cts, count, ids, rows, obj_asset, mass)
    assert np.array_equal(ref, mg) and np.array_equal(ref_f, mf) and np.array_equal(ref_st, rows)


def test_heavy_obstacles_approach_the_moving_solve():
    E = 400
    root, cts, count = random_contact_sets(E, 8)
    count, ids, obj_asset, rows, mass = random_bodies(root, cts, count, 58, kinematic=0.0)
    p = _full_params(iterations=6, friction=0.8)
    heavy = mass.copy()
    heavy[..., 0] = 1e-9
    heavy[..., 4:13] = (np.eye(3).reshape(9) * 1e-9)
    got, force, _, st = CD.solve(p, root, cts, count, ids, rows, obj_asset, heavy)
    u = CM.obstacle_point_velocity(rows, obj_asset, cts, ids)
    ref, ref_f, _ = CM.solve(p, root, cts, count, obstacle_velocity=u)
    scale = 1.0 + np.abs(root[:, 7:13]).max() + np.abs(rows[..., 7:13]).max()
    assert np.abs(got[:, 7:13] - ref[:, 7:13]).max() <= 1e-4 * scale
    assert np.abs(force - ref_f).max() <= 1e-4 * scale / float(p.dt)
    assert np.abs(st[..., 7:13] - rows[..., 7:13]).max() <= 1e-5  # the twist barely moves


def _momenta(p, root, rows, mass, free_assets):
    """total linear and angular momentum (about the world origin) of the robot and the given free assets, float64"""
    mr, cr, Jr = CD.robot_row_body(p)
    P, L = CD.body_momentum(root, mr, cr, Jr, origin_twist=False)
    for a in free_assets:
        m = 1.0 / float(mass[a, 0])
        pa, la = CD.body_momentum(rows[a], m, mass[a, 1:4], np.linalg.inv(mass[a, 4:13].astype(np.float64).reshape(3, 3)))
        P, L = P + pa, L + la
    return P, L


def test_momentum_is_conserved_without_the_ground():
    E = 200
    root, cts, count = random_contact_sets(E, 9)
    count, ids, obj_asset, rows, mass = random_bodies(root, cts, count, 59, kinematic=0.0, ground=False)
    p = _full_params(iterations=6, friction=1.0)
    got, _, _, st = CD.solve(p, root, cts, count, ids, rows, obj_asset, mass)
    after = rows.copy()
    after[..., 7:13] = st[..., 7:13]  # the solve's twists on the poses it ran with (the write-back's position correction aside)
    _, assets, nb = CD.gather_bodies(ids, count, obj_asset)
    checked = 0
    for e in range(E):
        if count[e] == 0:
            continue
        free = [int(a) for a in assets[e, :nb[e]]]
        P0, L0 = _momenta(p, root[e], rows[e], mass[e], free)
        P1, L1 = _momenta(p, got[e], after[e], mass[e], free)
        sP = 1.0 + np.abs(P0).max()
        sL = 1.0 + np.abs(L0).max() + 5.0 * sP
        assert np.abs(P1 - P0).max() <= 2e-5 * sP, (e, P0, P1)
        assert np.abs(L1 - L0).max() <= 2e-5 * sL, (e, L0, L1)
        checked += 1
    assert checked > 150


def _face_on(mr, mo, V, com_o=(0.0, 0.0, 0.0), inertia_o=np.eye(3), p_z=0.0):
    """a sphere (radius 0.2, mass mr, COM at its centre) at the origin moving at V along +x, touching a resting box whose face is
    at x = 0.2, with the depth at the rest offset (bias 0); the box origin at (0.7, 0, 0), the contact point at (0.2, 0, p_z)"""
    p = params(mass=mr, ground_plane=0, friction=0.5, iterations=4)
    root = np.zeros((1, 13), np.float32)
    root[0, 6], root[0, 7] = 1.0, V
    root[0, 2] = p_z
    cts = np.zeros((1, CMAX, 7), np.float32)
    cts[0, 0] = [0.2, 0.0, p_z, -1.0, 0.0, 0.0, p.rest_offset]
    rows = np.zeros((1, 1, 13), np.float32)
    rows[0, 0, 0], rows[0, 0, 6] = 0.7, 1.0
    mass = np.zeros((1, 1, 13), np.float32)
    mass[0, 0, 0], mass[0, 0, 1:4] = 1.0 / mo, com_o
    mass[0, 0, 4:13] = np.linalg.inv(np.asarray(inertia_o, np.float64)).reshape(9)
    ids = np.full((1, CMAX), -1, np.int32)
    ids[0, 0] = 0
    return p, root, cts, np.ones(1, np.int32), ids, rows, np.zeros((1, 1), np.int32), mass


@pytest.mark.parametrize("mr,mo", [(1.24, 1.0), (0.25, 1.0), (1.24, 0.1), (1.24, 13.0)])
def test_head_on_hit_ends_at_the_common_velocity(mr, mo):
    V = 3.0
    args = _face_on(mr, mo, V)
    got, force, _, st = CD.solve(*args)
    sg, sf, _, sst = shadow_dynamic(*args)
    assert np.array_equal(got, sg) and np.array_equal(st, sst)
    want = mr * V / (mr + mo)
    assert abs(got[0, 7] - want) <= 1e-6 * want and abs(st[0, 0, 7] - want) <= 1e-6 * want
    assert np.abs(got[0, 8:13]).max() == 0.0 and np.abs(st[0, 0, 8:13]).max() == 0.0
    # the force on the robot is its momentum change over dt; the box moved by dt x its velocity change
    p = args[0]
    assert abs(force[0, 0] - mr * (want - V) / p.dt) <= 1e-5 * mr * V / p.dt
    assert abs(st[0, 0, 0] - (0.7 + p.dt * want)) <= 1e-6


def test_kinetic_energy_never_rises_without_bias():
    E = 300
    root, cts, count = random_contact_sets(E, 10)
    cts[..., 6] = np.minimum(cts[..., 6], 0.001)  # depth <= rest_offset: no target separating velocity
    count, ids, obj_asset, rows, mass = random_bodies(root, cts, count, 60, kinematic=0.0)
    for friction in (0.0, 0.5, 2.0):
        p = _full_params(iterations=4, friction=friction)
        p.rest_offset = 0.001
        got, _, _, st = CD.solve(p, root, cts, count, ids, rows, obj_asset, mass)
        _, assets, nb = CD.gather_bodies(ids, count, obj_asset)
        mr, cr, Jr = CD.robot_row_body(p)
        for e in range(E):
            if count[e] == 0:
                continue
            e0, e1 = CD.body_energy(root[e], mr, cr, Jr, origin_twist=False), CD.body_energy(got[e], mr, cr, Jr, origin_twist=False)
            for a in assets[e, :nb[e]]:
                m, J = 1.0 / float(mass[e, a, 0]), np.linalg.inv(mass[e, a, 4:13].astype(np.float64).reshape(3, 3))
                after = rows[e, a].copy()
                after[7:13] = st[e, a, 7:13]
                e0 += CD.body_energy(rows[e, a], m, mass[e, a, 1:4], J)
                e1 += CD.body_energy(after, m, mass[e, a, 1:4], J)
            assert e1 <= e0 * (1 + 1e-5) + 1e-6, (friction, e, e0, e1)


def test_two_contacts_on_one_multi_part_asset_act_on_one_body():
    E = 300
    root, cts, count = random_contact_sets(E, 11)
    count, ids, obj_asset, rows, mass = random_bodies(root, cts, count, 61, kinematic=0.0, ground=False)
    one = np.zeros_like(obj_asset)  # every object a part of asset 0
    p = _full_params(iterations=6, friction=1.0)
    got, _, _, st = shadow_dynamic(p, root, cts, count, ids, rows, one, mass)
    ref, _, _, ref_st = CD.solve(p, root, cts, count, ids, rows, one, mass)
    assert np.array_equal(got, ref) and np.array_equal(st, ref_st)
    body, assets, nb = CD.gather_bodies(ids, count, one)
    assert nb.max() == 1 and (count > 1).sum() > 100
    assert np.array_equal(st[:, 1:], rows[:, 1:])  # only the one body is written
    after = rows.copy()
    after[..., 7:13] = st[..., 7:13]
    for e in np.nonzero(count > 1)[0][:80]:  # one body: the momentum balance counts its mass once
        P0, L0 = _momenta(p, root[e], rows[e], mass[e], [0])
        P1, L1 = _momenta(p, got[e], after[e], mass[e], [0])
        sP = 1.0 + np.abs(P0).max()
        assert np.abs(P1 - P0).max() <= 2e-5 * sP and np.abs(L1 - L0).max() <= 2e-5 * (1.0 + np.abs(L0).max() + 5.0 * sP)
    # as separate assets with the same rows the outcome differs
    sep = np.tile(np.arange(K_OBJ, dtype=np.int32) % A_AST, (E, 1))
    same = np.repeat(rows[:, :1], A_AST, axis=1)
    same_m = np.repeat(mass[:, :1], A_AST, axis=1)
    split, _, _, _ = CD.solve(p, root, cts, count, ids, same, sep, same_m)
    multi = count > 1
    assert not np.array_equal(split[multi, 7:13], ref[multi, 7:13])


def test_an_off_centre_hit_spins_a_tree_like_body():
    """13 kg with the COM 3 m above the base link, hit at the base level: the body turns about the horizontal axis, and the
    angular momentum about a fixed point is the robot's before"""
    mr, mo, V = 1.24, 13.0, 3.0
    J = np.diag([70.0, 90.0, 60.0])
    args = _face_on(mr, mo, V, com_o=(-0.5, 0.0, 3.0), inertia_o=J)
    got, _, _, st = CD.solve(*args)
    sg, _, _, sst = shadow_dynamic(*args)
    assert np.array_equal(got, sg) and np.array_equal(st, sst)
    p, root, rows, mass = args[0], args[1], args[5], args[7]
    assert st[0, 0, 11] < -1e-3 and abs(st[0, 0, 10]) < 1e-6 and abs(st[0, 0, 12]) < 1e-6  # pushed +x below the COM: w along -y
    after = rows.copy()
    after[..., 7:13] = st[..., 7:13]
    for about in ((0.0, 0.0, 0.0), (1.0, -2.0, 5.0)):
        mr_, cr, Jr = CD.robot_row_body(p)
        P0, L0 = CD.body_momentum(root[0], mr_, cr, Jr, about, origin_twist=False)
        P1, L1 = CD.body_momentum(got[0], mr_, cr, Jr, about, origin_twist=False)
        pa, la = CD.body_momentum(after[0, 0], mo, mass[0, 0, 1:4], J, about)
        assert np.abs(P1 + pa - P0).max() <= 1e-5 * mr * V
        assert np.abs(L1 + la - L0).max() <= 1e-5 * mr * V * 10.0
    # the hit transfers less momentum to a body that can turn than to one that only translates
    args_t = _face_on(mr, mo, V, com_o=(-0.5, 0.0, 0.0), inertia_o=J)
    got_t, _, _, _ = CD.solve(*args_t)
    assert got[0, 7] > got_t[0, 7]


def test_a_free_box_hit_by_a_sphere_keeps_moving():
    """the integrator: a sphere thrown at a resting 1 kg box pushes it off, and the pair's momentum is conserved throughout"""
    from tests.test_contact_moving_cpu import _box
    p = params(mass=1.24, ground_plane=0, friction=0.5, iterations=4)
    box = dict(tris=_box((0.4, 0.4, 0.4)), x=(0.6, 0.0, 0.0), mass=1.0, inertia=np.eye(3) * (1.0 * 0.32 / 12))
    h = CD.simulate_dynamic(p, (0.0, 0.0, 0.0), (3.0, 0.0, 0.0), (0.0, 0.0, 0.0), 40, [box])
    hit = np.nonzero(np.linalg.norm(h["force"], axis=1) > 0)[0]
    assert len(hit) > 0
    vb = h["rows"][-1, 0, 7]
    assert vb > 1.0 and h["rows"][-1, 0, 0] > 0.6 + 0.5 * vb * p.dt * (40 - hit[0]) * 0.5
    P = 1.24 * h["root"][:, 7].astype(np.float64) + 1.0 * h["rows"][:, 0, 7].astype(np.float64)
    assert np.abs(P - 1.24 * 3.0).max() <= 1e-4 * 3.0
    assert h["root"][-1, 7] <= vb + 1e-5  # the robot does not pass the box


def test_argument_validation(tmp_path):
    from aerial_gym_simulator_b200 import urdf
    from aerial_gym_simulator_b200.env_manager import EnvManager
    from aerial_gym_simulator_b200.env_manager.env_manager import _obstacle_mass_row
    from aerial_gym_simulator_b200.hp2 import ContactMotion, ObstacleMass, contact

    for bad in ({"contact": "rigid", "contact_dynamic_obstacles": True},
                {"contact": "rigid", "contact_moving_obstacles": False, "contact_dynamic_obstacles": True},
                {"contact": "rigid", "contact_moving_obstacles": True, "contact_dynamic_obstacles": 1},
                {"contact": "rigid", "contact_moving_obstacles": True, "contact_dynamic_obstacles": "yes"}):
        with pytest.raises(ValueError, match="contact_dynamic_obstacles"):
            EnvManager("base_sim", "dynamic_env", "base_quadrotor", "lee_velocity_control", "cpu", args=bad, num_envs=2)
    with pytest.raises(ValueError, match="contact_moving_obstacles"):
        EnvManager("base_sim", "dynamic_env", "base_quadrotor", "lee_velocity_control", "cpu",
                   args={"contact_moving_obstacles": True, "contact_dynamic_obstacles": True}, num_envs=2)
    # a URDF without inertials: no density is guessed, the error names the file
    f = tmp_path / "massless.urdf"
    f.write_text('<robot name="m"><link name="base"><visual><geometry><box size="1 1 1"/></geometry></visual></link></robot>')
    with pytest.raises(ValueError, match="massless.urdf"):
        _obstacle_mass_row(urdf.parse_urdf(str(f)), str(f))
    from aerial_gym_simulator_b200.config import asset_config as ac
    row = _obstacle_mass_row(urdf.parse_urdf(f"{ac._ENV_ASSETS}/objects/1_x_1_wall.urdf"), "1_x_1_wall.urdf")
    assert row.dtype == np.float32 and row[0] == 1.0 and np.array_equal(row[4:], np.eye(3, dtype=np.float32).reshape(9))
    # the mass table holder
    E, A, K = 3, 4, 5
    t = torch.zeros(E, A, 13)
    t[..., 0] = 1.0
    m = ObstacleMass(t)
    assert (m.E, m.A) == (E, A)
    for bad in (t.double(), torch.zeros(E, A, 12), torch.zeros(E, 13), torch.zeros(E, 0, 13), torch.zeros(E, 13, A).transpose(1, 2),
                torch.full((E, A, 13), float("nan")), torch.full((E, A, 13), float("inf")), -t):
        with pytest.raises(ValueError):
            ObstacleMass(bad)
    st, oa = torch.zeros(E, A, 13), torch.randint(0, A, (E, K), dtype=torch.int32)
    mo = ContactMotion(st, oa)
    rs, f_, cr = torch.zeros(E, 13), torch.zeros(E, 3), torch.zeros(E, dtype=torch.bool)
    with pytest.raises(_lib.AgxError, match="CUDA"):
        contact(None, rs, params(), f_, cr, motion=mo, mass=m)
    lib = _lib.load()
    assert lib.agx_sizeof(13) == C.sizeof(_lib.AgxObstacleMass) == 52
    # the C entry point refuses a NULL scene, and a NULL mass table before it looks at anything else
    assert lib.agx_hp2_contact_dynamic(None, 0, C.byref(params()), C.byref(mo.c), C.c_void_p(t.data_ptr()), None, 13, None, None, None,
                                       None) == -3
    assert lib.agx_hp2_contact_dynamic(C.byref(_lib.AgxHp2Scene()), 0, C.byref(params()), C.byref(mo.c), None, None, 13, None, None,
                                       None, None) == -3
