"""Rigid contact mode on the CPU: the solve of contact_core.cuh (compiled for the host) against oracle/contact_oracle.py bit for bit,
the contact selection order, argument checks, and the physics of the model on a free sphere integrated by the oracle."""
import ctypes as C

import numpy as np
import pytest
import torch

from aerial_gym_simulator_b200 import _lib
from oracle import contact_oracle as CO
from oracle import hp2_oracle as RO
from tests import _contact_shadow

_p = lambda a: C.c_void_p(a.ctypes.data)


def params(**kw):
    p = _lib.AgxContactParams()
    d = dict(radius=0.2, contact_offset=0.002, rest_offset=0.001, dt=0.01, mass=1.0, friction=1.0, max_depenetration_velocity=1.0,
             force_threshold=0.05, iterations=4, ground_plane=1)
    d.update(kw)
    inertia_inv = d.pop("inertia_inv", None)
    if inertia_inv is None:  # solid sphere of the given radius and mass
        inertia_inv = np.eye(3) / (0.4 * d["mass"] * d["radius"] ** 2)
    com = d.pop("com", (0.0, 0.0, 0.0))
    for k, v in d.items():
        setattr(p, k, v)
    p.inertia_inv[:] = [float(v) for v in np.asarray(inertia_inv, np.float32).reshape(9)]
    p.com[:] = [float(v) for v in com]
    return p


def random_contact_sets(E, seed):
    g = np.random.default_rng(seed)
    root = np.zeros((E, 13), np.float32)
    root[:, 0:3] = g.uniform(-3, 3, (E, 3))
    q = g.normal(size=(E, 4))
    root[:, 3:7] = q / np.linalg.norm(q, axis=1, keepdims=True)
    root[:, 7:13] = g.normal(size=(E, 6)) * 2.0
    count = g.integers(0, CO.CONTACT_MAX + 1, E).astype(np.int32)
    n = g.normal(size=(E, CO.CONTACT_MAX, 3))
    n /= np.linalg.norm(n, axis=2, keepdims=True)
    depth = g.uniform(-0.002, 0.08, (E, CO.CONTACT_MAX))
    cts = np.zeros((E, CO.CONTACT_MAX, 7), np.float32)
    cts[..., 0:3] = root[:, None, 0:3] - n * (0.2 - depth)[..., None]
    cts[..., 3:6], cts[..., 6] = n, depth
    return root, cts, count


@pytest.mark.parametrize("iterations,friction,seed", [(1, 0.0, 0), (4, 1.0, 1), (10, 0.5, 2), (4, 2.0, 3)])
def test_shadow_solve_matches_oracle_bit_for_bit(iterations, friction, seed):
    E = 600
    root, cts, count = random_contact_sets(E, seed)
    ii = np.array([[40.0, 1.5, -0.7], [1.5, 35.0, 0.3], [-0.7, 0.3, 22.0]])  # a full symmetric inverse inertia
    p = params(iterations=iterations, friction=friction, mass=1.2, inertia_inv=ii, com=(0.01, -0.02, 0.005), force_threshold=60.0)
    got = root.copy()
    force = np.zeros((E, 3), np.float32)
    crash = np.zeros(E, np.uint8)
    _contact_shadow.load().shadow_contact_solve(E, C.byref(p), _p(got), 13, _p(cts), _p(count), _p(force), _p(crash))
    ref, ref_f, ref_c = CO.solve(p, root, cts, count)
    assert np.array_equal(got, ref), f"{(got != ref).sum()} state values differ"
    assert np.array_equal(force, ref_f)
    assert np.array_equal(crash.astype(bool), ref_c)
    assert 0 < ref_c.sum() < (count > 0).sum()
    assert not np.array_equal(got[:, 7:13], root[:, 7:13])


def test_selection_keeps_the_nearest_by_distance_then_index():
    g = np.random.default_rng(5)
    sel = _contact_shadow.load().shadow_contact_select
    for trial in range(200):
        n = int(g.integers(0, 20))
        key = g.choice(np.array([-0.01, 0.0, 0.05, 0.1, 0.15], np.float32), n).astype(np.float32)  # many ties
        obj = g.permutation(n).astype(np.int32)
        out = np.zeros(CO.CONTACT_MAX, np.int32)
        k = sel(n, _p(key), _p(obj), _p(out))
        want = [int(o) for _, o in sorted(zip(key.tolist(), obj.tolist()))][:CO.CONTACT_MAX]
        assert k == len(want) and out[:k].tolist() == want


def test_argument_validation():
    from aerial_gym_simulator_b200.env_manager import EnvManager
    from aerial_gym_simulator_b200.hp2 import contact

    for bad in ({"contact": "soft"}, {"contact": True}, {"contact_friction": -0.1}, {"contact_friction": float("nan")},
                {"contact_friction": "1"}, {"contact_friction": True}):
        with pytest.raises(ValueError):
            EnvManager("base_sim", "env_with_obstacles", "base_quadrotor", "lee_velocity_control", "cpu", args=bad, num_envs=2)
    E = 4
    rs, f, cr = torch.zeros(E, 13), torch.zeros(E, 3), torch.zeros(E, dtype=torch.bool)
    with pytest.raises(_lib.AgxError, match="CUDA"):
        contact(None, rs, params(), f, cr)
    assert _lib.load().agx_sizeof(11) == C.sizeof(_lib.AgxContactParams)


def _box_wall(size, centre):
    t = RO.box_template(size).reshape(-1, 3, 3) + np.asarray(centre, np.float32)
    return np.concatenate([t[:, 0], t[:, 1] - t[:, 0], t[:, 2] - t[:, 0]], axis=1).astype(np.float32)


def _energy(p, h, z0=0.0):
    m = float(p.mass)
    I = np.linalg.inv(np.asarray(p.inertia_inv, np.float64).reshape(3, 3))
    v, w = h["v"].astype(np.float64), h["w"].astype(np.float64)
    return 0.5 * m * (v ** 2).sum(1) + 0.5 * np.einsum("si,ij,sj->s", w, I, w) + m * 9.81 * (h["x"][:, 2].astype(np.float64) - z0)


def _energy_never_rises(e):
    # the state is float32: allow its rounding (1e-6 of the energy's scale) and nothing more
    assert np.diff(e).max() <= 1e-6 * np.abs(e).max(), f"energy rises by {np.diff(e).max()}"


def test_dropped_sphere_comes_to_rest_on_the_ground():
    p = params()
    h = CO.simulate(p, (0.0, 0.0, 1.0), (0.0, 0.0, 0.0), (0.0, 0.0, 0.0), 500)
    depth = p.radius - h["x"][:, 2]
    # at rest the integrator's gravity re-penetrates g dt^2 ~ 1 mm per sub-step, the solve's separating velocity takes it back
    assert depth[-1] <= p.rest_offset + 0.002 and depth.max() < p.radius
    assert np.abs(h["v_pre"][-1]).max() < 1e-2
    assert np.abs(h["x"][-1] - h["x"][-2]).max() / p.dt < 1e-2
    assert h["force"][-1][2] == pytest.approx(p.mass * 9.81, rel=0.01)  # it carries its weight
    _energy_never_rises(_energy(p, h))


def test_sphere_thrown_into_a_wall_never_crosses_its_face():
    p = params()
    wall = _box_wall((0.2, 4.0, 4.0), (1.0, 0.0, 1.0))  # face plane x = 0.9
    h = CO.simulate(p, (0.0, 0.0, 1.0), (5.0, 0.0, 0.0), (0.0, 0.0, 0.0), 500, objects=[wall])
    assert h["x"][:, 0].max() < 0.9
    assert h["x"][:, 0].max() > 0.9 - p.radius  # it did reach the wall
    assert (h["v"][:, 0] <= 1e-6).all() or h["x"][-1, 0] < 0.9 - p.radius  # stopped or bounced off, never pushed in
    _energy_never_rises(_energy(p, h))


def test_sliding_stops_within_the_coulomb_distance():
    v0, mu = 4.0, 1.0
    p = params(friction=mu, inertia_inv=np.zeros((3, 3)))  # a slider that cannot roll
    h = CO.simulate(p, (0.0, 0.0, p.radius - p.rest_offset), (v0, 0.0, 0.0), (0.0, 0.0, 0.0), 500)
    assert np.abs(h["v"][-1, 0:2]).max() < 1e-3
    want = v0 ** 2 / (2 * mu * 9.81)
    assert h["x"][-1, 0] == pytest.approx(want, rel=0.05)
    m = float(p.mass)
    e = 0.5 * m * (h["v"].astype(np.float64) ** 2).sum(1) + m * 9.81 * h["x"][:, 2].astype(np.float64)
    _energy_never_rises(e)
