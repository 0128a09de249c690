"""Rigid contact with moving obstacles on the CPU: the MOVING solve of contact_core.cuh (compiled for the host) against
oracle/contact_moving_oracle.py bit for bit, its reduction to the static solve at u = 0, the Galilean invariance of the model, the
physics of a free sphere among moving obstacles, and the argument checks."""
import ctypes as C

import numpy as np
import pytest
import torch

from aerial_gym_simulator_b200 import _lib
from oracle import contact_moving_oracle as CM
from oracle import contact_oracle as CO
from oracle import hp2_oracle as RO
from tests import _contact_moving_shadow, _contact_shadow
from tests.test_contact_cpu import _energy_never_rises, params, random_contact_sets

_p = lambda a: C.c_void_p(a.ctypes.data)
G = 9.81


def random_twists(cts, seed):
    """asset rows for every contact slot (one asset per contact): a centre within 1 m of the contact point, |v| <= 3 m/s,
    |w| <= 2 rad/s; ids map slot i to asset i"""
    E = cts.shape[0]
    g = np.random.default_rng(seed)
    rows = np.zeros((E, CO.CONTACT_MAX, 13), np.float32)
    rows[..., 0:3] = cts[..., 0:3] + g.uniform(-1, 1, (E, CO.CONTACT_MAX, 3))
    rows[..., 6] = 1.0
    d = g.normal(size=(E, CO.CONTACT_MAX, 6))
    rows[..., 7:10] = d[..., 0:3] / np.linalg.norm(d[..., 0:3], axis=-1, keepdims=True) * g.uniform(0, 3, (E, CO.CONTACT_MAX, 1))
    rows[..., 10:13] = d[..., 3:6] / np.linalg.norm(d[..., 3:6], axis=-1, keepdims=True) * g.uniform(0, 2, (E, CO.CONTACT_MAX, 1))
    obj_asset = np.tile(np.arange(CO.CONTACT_MAX, dtype=np.int32), (E, 1))
    return rows, obj_asset


def shadow_moving(p, root, cts, count, u):
    got = root.copy()
    force = np.zeros((root.shape[0], 3), np.float32)
    crash = np.zeros(root.shape[0], np.uint8)
    _contact_moving_shadow.load().shadow_contact_solve_moving(root.shape[0], C.byref(p), _p(got), 13, _p(cts), _p(count),
                                                              _p(np.ascontiguousarray(u, np.float32)), _p(force), _p(crash))
    return got, force, crash.astype(bool)


def _full_params(**kw):
    ii = np.array([[40.0, 1.5, -0.7], [1.5, 35.0, 0.3], [-0.7, 0.3, 22.0]])  # a full symmetric inverse inertia
    d = dict(mass=1.2, inertia_inv=ii, com=(0.01, -0.02, 0.005), force_threshold=60.0)
    d.update(kw)
    return params(**d)


@pytest.mark.parametrize("iterations,friction,seed", [(1, 0.0, 0), (4, 1.0, 1), (10, 0.5, 2), (4, 2.0, 3)])
def test_shadow_moving_solve_matches_oracle_bit_for_bit(iterations, friction, seed):
    E = 600
    root, cts, count = random_contact_sets(E, seed)
    rows, obj_asset = random_twists(cts, seed + 100)
    ids = np.where(np.arange(CO.CONTACT_MAX)[None] < count[:, None], np.arange(CO.CONTACT_MAX)[None], -1).astype(np.int32)
    u = CM.obstacle_point_velocity(rows, obj_asset, cts, ids)
    # the kernel's u, through the header's own function
    su = np.zeros(3, np.float32)
    for e in range(0, E, 7):
        for i in range(count[e]):
            _contact_moving_shadow.load().shadow_obstacle_point_vel(_p(rows[e, i]), _p(np.ascontiguousarray(cts[e, i, 0:3])), _p(su))
            assert np.array_equal(su, u[e, i])
    assert np.abs(u[count > 0]).max() > 1.0
    p = _full_params(iterations=iterations, friction=friction)
    got, force, crash = shadow_moving(p, root, cts, count, u)
    ref, ref_f, ref_c = CM.solve(p, root, cts, count, obstacle_velocity=u)
    assert np.array_equal(got, ref), f"{(got != ref).sum()} state values differ"
    assert np.array_equal(force, ref_f)
    assert np.array_equal(crash, ref_c)
    static, _, _ = CO.solve(p, root, cts, count)
    assert not np.array_equal(ref[:, 7:13], static[:, 7:13])  # the obstacle velocities do enter


def test_zero_obstacle_velocity_is_the_static_solve():
    E = 600
    root, cts, count = random_contact_sets(E, 7)
    p = _full_params(iterations=4, friction=1.0)
    got, force, crash = shadow_moving(p, root, cts, count, np.zeros((E, CO.CONTACT_MAX, 3), np.float32))
    st = root.copy()
    sf = np.zeros((E, 3), np.float32)
    sc = np.zeros(E, np.uint8)
    _contact_shadow.load().shadow_contact_solve(E, C.byref(p), _p(st), 13, _p(cts), _p(count), _p(sf), _p(sc))
    assert np.array_equal(got, st) and np.array_equal(force, sf) and np.array_equal(crash, sc.astype(bool))
    ref, ref_f, ref_c = CM.solve(p, root, cts, count, obstacle_velocity=np.zeros((E, CO.CONTACT_MAX, 3), np.float32))
    assert np.array_equal(ref, st) and np.array_equal(ref_f, sf)


def test_galilean_invariance():
    """a uniform obstacle velocity u = the static problem in the frame moving with u, shifted back"""
    E = 400
    root, cts, count = random_contact_sets(E, 8)
    p = _full_params(iterations=6, friction=0.8)
    g = np.random.default_rng(9)
    ue = g.uniform(-3, 3, (E, 3)).astype(np.float32)
    u = np.repeat(ue[:, None, :], CO.CONTACT_MAX, axis=1)
    got, f, c = CM.solve(p, root, cts, count, obstacle_velocity=u)
    moved = root.copy()
    moved[:, 7:10] -= ue
    ref, ref_f, _ = CO.solve(p, moved, cts, count)
    ref[:, 7:10] += ue
    scale = 1.0 + np.abs(root[:, 7:13]).max() + np.abs(ue).max()
    assert np.abs(got[:, 7:13] - ref[:, 7:13]).max() <= 1e-5 * scale
    assert np.abs(f - ref_f).max() <= 1e-5 * scale / float(p.dt)


def _box(size, centre=(0.0, 0.0, 0.0)):
    t = RO.box_template(size).reshape(-1, 3, 3) + np.asarray(centre, np.float32)
    return np.concatenate([t[:, 0], t[:, 1] - t[:, 0], t[:, 2] - t[:, 0]], axis=1).astype(np.float32)


def test_a_moving_wall_pushes_a_free_sphere():
    p = params(ground_plane=0)
    u = 2.0
    # wall face at x = -0.3 moving +x towards a sphere at rest at the origin, 2 m up so that it stays clear of nothing else
    wall = dict(tris=_box((0.2, 4.0, 4.0)), x=(-0.4, 0.0, 2.0), v=(u, 0.0, 0.0))
    h = CM.simulate_moving(p, (0.0, 0.0, 2.0), (0.0, 0.0, 0.0), (0.0, 0.0, 0.0), 60, [wall])
    hit = np.nonzero(np.linalg.norm(h["force"], axis=1) > 0)[0]
    assert len(hit) > 0
    assert h["v"][hit[0]:, 0].min() >= u * (1 - 1e-5)  # after the impact the sphere never moves slower than the wall
    bound = p.rest_offset + u * p.dt + G * p.dt ** 2
    assert h["depth"].max() <= bound + 1e-5, f"penetration {h['depth'].max()} > {bound}"
    m = float(p.mass)  # kinetic energy in the wall's frame
    e = 0.5 * m * ((h["v"].astype(np.float64) - [u, 0.0, 0.0]) ** 2).sum(1) + m * G * h["x"][:, 2].astype(np.float64)
    _energy_never_rises(e[hit[0]:])


def test_a_sliding_platform_carries_a_sphere_at_the_coulomb_rate():
    mu, u = 1.0, 1.0
    p = params(friction=mu, inertia_inv=np.zeros((3, 3)), ground_plane=0)  # a slider that cannot roll
    plat = dict(tris=_box((40.0, 40.0, 0.2)), x=(0.0, 0.0, -0.1), v=(u, 0.0, 0.0))  # top face z = 0
    h = CM.simulate_moving(p, (0.0, 0.0, p.radius - p.rest_offset), (0.0, 0.0, 0.0), (0.0, 0.0, 0.0), 60, [plat])
    vx = h["v"][:, 0].astype(np.float64)
    slip = np.nonzero(vx < u - 1e-3)[0]
    assert len(slip) >= 5
    rate = np.diff(vx[: slip[-1] + 1]) / p.dt
    assert np.abs(rate[1:] - mu * G).max() <= 0.05 * mu * G, rate
    assert np.abs(vx[-10:] - u).max() < 1e-4  # it then rides along
    assert np.abs(h["v"][-10:, 1]).max() < 1e-6
    m = float(p.mass)
    e = 0.5 * m * ((h["v"].astype(np.float64) - [u, 0.0, 0.0]) ** 2).sum(1) + m * G * h["x"][:, 2].astype(np.float64)
    _energy_never_rises(e)


def test_a_turntable_carries_a_sphere_at_w_cross_r():
    wz = 1.0
    p = params(friction=1.0, inertia_inv=np.zeros((3, 3)), ground_plane=0)
    table = dict(tris=_box((6.0, 6.0, 0.2), (0.0, 0.0, -0.1)), x=(0.0, 0.0, 0.0), v=(0.0, 0.0, 0.0), wz=wz)
    h = CM.simulate_moving(p, (1.0, 0.0, p.radius - p.rest_offset), (0.0, 0.0, 0.0), (0.0, 0.0, 0.0), 300, [table])
    x, v = h["x"][-50:].astype(np.float64), h["v"][-50:].astype(np.float64)
    want = np.stack([-wz * x[:, 1], wz * x[:, 0]], axis=1)
    assert np.abs(v[:, 0:2] - want).max() < 0.02 * wz
    r = np.linalg.norm(h["x"][:, 0:2], axis=1)
    assert np.abs(r - 1.0).max() < 0.05  # friction holds it on its circle


def test_argument_validation():
    from aerial_gym_simulator_b200.env_manager import EnvManager
    from aerial_gym_simulator_b200.hp2 import ContactMotion, contact

    for bad in ({"contact_moving_obstacles": True}, {"contact": "flag", "contact_moving_obstacles": True},
                {"contact": "rigid", "contact_moving_obstacles": 1}, {"contact": "rigid", "contact_moving_obstacles": "yes"}):
        with pytest.raises(ValueError, match="contact_moving_obstacles"):
            EnvManager("base_sim", "dynamic_env", "base_quadrotor", "lee_velocity_control", "cpu", args=bad, num_envs=2)
    E, A, K = 3, 4, 5
    st, oa = torch.zeros(E, A, 13), torch.randint(0, A, (E, K), dtype=torch.int32)
    m = ContactMotion(st, oa)
    assert m.c.asset_stride == 13 and m.c.num_assets == A and m.obj_asset.dtype == torch.int32
    assert ContactMotion(torch.zeros(E, A, 16)[..., :13], oa.long()).c.asset_stride == 16  # a view with wider rows
    for bad_st, bad_oa in ((st.double(), oa), (torch.zeros(E, A, 12), oa), (torch.zeros(E, 13), oa), (torch.zeros(E, 0, 13), oa),
                           (torch.zeros(E, 13, A).transpose(1, 2), oa), (st, oa.float()), (st, oa[:2]), (st, oa[0]),
                           (st, oa + A), (st, oa - A)):
        with pytest.raises(ValueError):
            ContactMotion(bad_st, bad_oa)
    rs, f, cr = torch.zeros(E, 13), torch.zeros(E, 3), torch.zeros(E, dtype=torch.bool)
    with pytest.raises(_lib.AgxError, match="CUDA"):
        contact(None, rs, params(), f, cr, motion=m)
    assert _lib.load().agx_sizeof(12) == C.sizeof(_lib.AgxContactMotion)
    lib = _lib.load()
    # the C entry point refuses a NULL scene and a bad motion before it looks at anything else
    assert lib.agx_hp2_contact_moving(None, 0, C.byref(params()), C.byref(m.c), None, 13, None, None, None, None) == -3
