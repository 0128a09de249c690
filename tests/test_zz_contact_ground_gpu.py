"""Obstacle-ground contact (args['contact_obstacle_ground'], agx_obstacle_ground_contact) on the GPU: the kernel against
oracle/contact_ground_oracle.py in dynamic_env and on sphere and box hulls; objects driven into the floor stop at it and objects that
start under it rise, while without the key they sink; a robot pushing an object into the floor; no change where nothing nears the
ground; graph and launch step modes bit-identical."""
import random

import numpy as np
import pytest
import torch

from aerial_gym_simulator_b200 import _lib
from aerial_gym_simulator_b200.hp2 import (ContactMotion, ObstacleHull, ObstacleMass, box_triangles, icosphere_triangles,
                                           obstacle_ground_contact)
from oracle import contact_ground_oracle as CG
from tests.test_zz_contact_gpu import _env
from tests.test_zz_contact_moving_gpu import _moving_test_env, _place, _twists, random_twists

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GROUND = dict(contact_moving_obstacles=True, contact_dynamic_obstacles=True, contact_obstacle_ground=True)
DYN = dict(contact_moving_obstacles=True, contact_dynamic_obstacles=True)


@pytest.fixture(autouse=True)
def _needs_the_kernels():
    if DEV == "cpu":  # the CPU dry run of the GPU test text: the contact kernels have no CPU twin
        pytest.skip("the contact kernels have no CPU twin")


def _tables(hull):
    return (hull.vertices.cpu().numpy(), hull.file_offset.cpu().numpy(), hull.file_reach.cpu().numpy(),
            hull.asset_file.cpu().numpy().reshape(-1))


def check_ground_against_oracle(p, st, mass, hull):
    """one launch on rows st [E,A,13] (a CPU tensor) against the oracle, with test_zz_contact_dynamic_gpu's tolerances; rows with a
    vertex within float rounding of contact_offset are left out.  Returns the oracle's count per row."""
    E, A = st.shape[:2]
    rows = st.to(DEV).contiguous()
    obstacle_ground_contact(p, ContactMotion(rows, torch.zeros(E, 1, dtype=torch.int32, device=DEV)), mass, hull)
    torch.cuda.synchronize()
    v, off, reach, af = _tables(hull)
    r0, m = st.numpy().reshape(E * A, 13), mass.table.cpu().numpy().reshape(E * A, 13)
    ref, _, count = CG.ground_contact(p, r0, m, v, off, reach, af)
    got = rows.cpu().numpy().reshape(E * A, 13)
    # rows with a vertex whose height is within float rounding of contact_offset: whether it is a candidate is arbitrary
    amb = np.zeros(E * A, bool)
    for f in np.unique(af):
        sel = np.nonzero(af == f)[0]
        z = np.stack(CG._world(r0[sel].astype(np.float64), v[off[f]:off[f + 1]].astype(np.float64)))[2]
        amb[sel] = (np.abs(z - p.contact_offset) <= 1e-6 * (1.0 + np.abs(r0[sel, 2:3]))).any(axis=1)
    ok = ~amb
    assert amb.mean() < 0.01
    touched_gpu, touched_ref = (got != r0).any(axis=1), (ref != r0).any(axis=1)
    assert np.array_equal(touched_gpu[ok], touched_ref[ok]), "touched rows differ"
    vs = 1.0 + np.abs(r0[:, 7:13]).max() * 10.0
    assert (np.abs(got[ok, 7:13] - ref[ok, 7:13]) <= 5e-3 * (vs + np.abs(ref[ok, 7:13]))).all(), \
        f"max velocity error {np.abs(got[ok, 7:13] - ref[ok, 7:13]).max()}"
    assert (np.abs(got[ok, 0:7] - ref[ok, 0:7]) <= 1e-4 * (1.0 + np.abs(ref[ok, 0:7]))).all(), "poses differ"
    return count


def test_ground_kernel_matches_oracle_in_dynamic_env():
    env = _env("dynamic_env", n=77, seed=40, **GROUND)
    assert (env.num_envs * env.num_obs_in_env) % 32 != 0
    p, mass, hull = env.contact_params, env._obstacle_mass, env._obstacle_hull
    assert hull.F == 4 and hull.vertices.shape[0] == 32  # the four box files of objects/, 8 vertices each
    st = random_twists(env.global_tensor_dict["env_asset_state_tensor"].cpu(), seed=41)
    g = torch.Generator().manual_seed(42)
    st[..., 2] = torch.rand(st.shape[:2], generator=g) * 2.5 - 1.0  # straddling the ground
    count = check_ground_against_oracle(p, st, mass, hull)
    assert 0.2 < (count > 0).mean() < 0.9 and (count == 8).any()


def test_ground_kernel_matches_oracle_on_sphere_and_box_hulls():
    E, A = 45, 7
    files = [np.unique(icosphere_triangles(0.3).reshape(-1, 3), axis=0), np.unique(box_triangles((0.5, 0.2, 1.0)).reshape(-1, 3), axis=0)]
    g = np.random.default_rng(43)
    hull = ObstacleHull.from_files(files, g.integers(0, 2, (E, A)), DEV)
    st = torch.zeros(E, A, 13)
    st[..., 0:2] = torch.from_numpy(g.uniform(-3, 3, (E, A, 2)).astype(np.float32))
    st[..., 2] = torch.from_numpy(g.uniform(-0.8, 1.0, (E, A)).astype(np.float32))
    q = torch.from_numpy(g.normal(size=(E, A, 4)).astype(np.float32))
    st[..., 3:7] = q / q.norm(dim=-1, keepdim=True)
    st = random_twists(st, seed=44)
    m = np.zeros((E, A, 13), np.float32)
    m[..., 0] = 1.0 / g.uniform(0.2, 5.0, (E, A))
    m[..., 1:4] = g.uniform(-0.1, 0.1, (E, A, 3))
    m[..., 4:13] = (np.eye(3) * 20.0).reshape(9)
    m[g.uniform(size=(E, A)) < 0.1] = 0.0  # kinematic rows
    mass = ObstacleMass(torch.from_numpy(m).to(DEV))
    p = _lib.AgxContactParams(contact_offset=0.002, rest_offset=0.001, dt=0.01, friction=0.7, max_depenetration_velocity=1.0,
                                 iterations=6)
    count = check_ground_against_oracle(p, st, mass, hull)
    assert (count == 8).mean() > 0.2 and not count[m.reshape(E * A, 13).any(axis=1) == 0].any()


def _lowest(env, tables=None):
    """lowest world vertex height of every (env, asset) row [E,A]; tables: _tables() of a hull of the same assets (default: the
    env's own)"""
    st = env.global_tensor_dict["env_asset_state_tensor"].cpu().numpy()
    E, A = st.shape[:2]
    v, off, _, af = tables if tables is not None else _tables(env._obstacle_hull)
    return CG.lowest_vertex(st.reshape(E * A, 13), v, off, af).reshape(E, A)


def _push_down(env, g):
    tw = torch.zeros(env.num_envs, env.num_obs_in_env, 6, device=DEV)
    tw[..., 2] = -torch.rand(env.num_envs, env.num_obs_in_env, generator=g, device=DEV) * 2.0
    return tw


def _sink_run(ground, tables=None, steps=50, n=300):
    """50 env steps of dynamic_env with every object pushed down at up to 2 m/s; the same seed selects the same assets with and
    without the key, so the run without it is measured with the tables of the run with it"""
    env = _env("dynamic_env", n=n, seed=45, **(GROUND if ground else DYN))
    tables = tables if tables is not None else _tables(env._obstacle_hull)
    act = torch.zeros(env.num_envs, env.num_robot_actions, device=DEV)
    g = torch.Generator(device=DEV).manual_seed(46)
    ast = env.global_tensor_dict["env_asset_state_tensor"]
    active = (ast[..., 2] > -500.0).cpu().numpy()  # parked assets (z = -1000) are out of play
    low0 = _lowest(env, tables)
    lows = []
    for step in range(steps):
        random.seed(600 + step)
        env.step(actions=act, env_actions=_push_down(env, g))
        lows.append(_lowest(env, tables))
    torch.cuda.synchronize()
    return env, tables, active, low0, np.asarray(lows)


def test_objects_pushed_down_stop_at_the_ground_and_buried_ones_rise():
    env, tables, active, low0, lows = _sink_run(True)
    p = env.contact_params
    per_step = env.cfg.env.num_physics_steps_per_env_step_mean * p.dt
    after = int(np.ceil(1.0 / per_step))  # the first second
    bound = p.rest_offset + 2.0 * p.dt * 2.0
    assert (low0[active] < -0.05).sum() > 50  # objects start under the floor ...
    worst = lows[after:][:, active].min()
    assert worst >= -bound, f"an active object's lowest vertex at {worst:.4f} m < -{bound:.4f} m"
    # ... and most are on it at the end (the solve's position correction leaves them up to one sub-step of travel above it)
    assert (lows[-1][active] < bound + p.contact_offset).mean() > 0.5
    # without the key the same run puts them well below the floor
    _, _, active_off, _, lows_off = _sink_run(False, tables)
    assert np.array_equal(active, active_off)
    assert lows_off[-1][active].min() < -2.0 and (lows_off[-1][active] < -bound).mean() > 0.5


def test_a_robot_pushing_an_object_into_the_floor_leaves_it_on_the_floor():
    env = _moving_test_env("contact_ground_push_test_env", "objects", "small_cube.urdf", n=37, seed=47, controller="no_control",
                           contact_dynamic_obstacles=True, contact_obstacle_ground=True)  # 0.4 m cube, 1 kg
    p, R = env.contact_params, env.robot.collision_radius
    ast = env.global_tensor_dict["env_asset_state_tensor"]
    _place(env, (0.0, 0.0, 0.2 + 0.2 + R + 0.01), (0.0, 0.0, 0.2))  # the cube on the floor, the robot 1 cm above it
    env.engine.root_state[:, 9] = -3.0
    env.cfg.env.num_physics_steps_per_env_step_mean = 1  # one sub-step per env step: the force and the flag of each sub-step
    act = torch.zeros(env.num_envs, env.num_robot_actions, device=DEV)
    pushed = False
    for step in range(60):
        env.reset_tensors()
        env.step(actions=act)
        torch.cuda.synchronize()
        f = env.global_tensor_dict["robot_contact_force_tensor"]
        assert torch.equal(env.collision_tensor, f.norm(dim=1) > p.force_threshold), f"step {step}: crash flag != force rule"
        low = _lowest(env)[:, 0]
        # the robot's solve runs after the ground's: the cube may end the sub-step below the ground by dt |dv| of that solve, and
        # the largest |dv| a 1.24 kg robot at 3 m/s gives a 1 kg cube is 2 m_r V / (m_r + m_o) < 2 V
        allowance = p.rest_offset + p.contact_offset + p.dt * 2.0 * 3.0
        assert (low >= -allowance).all(), (step, float(low.min()))
        pushed |= bool((f.norm(dim=1) > 0).any())
    assert pushed
    low = _lowest(env)[:, 0]
    assert np.abs(low).max() < 0.03 and bool((ast[:, 0, 2] > 0.17).all())  # on the floor, not under it
    assert bool((env.engine.root_state[:, 2] > 0.4).all())  # and the robot on top of it


def _high_env(ground, n=61, seed=48):
    from aerial_gym_simulator_b200.config.env_config import DynamicEnvironmentCfg as base
    from aerial_gym_simulator_b200.registry._core import env_config_registry

    class High(base):
        class env(base.env):
            lower_bound_min = [-2.0, -4.0, 10.0]
            lower_bound_max = [-1.0, -2.5, 10.0]
            upper_bound_min = [9.0, 2.5, 14.0]
            upper_bound_max = [10.0, 4.0, 15.0]
    env_config_registry.register("contact_ground_high_test_env", High)
    env = _env("contact_ground_high_test_env", n=n, seed=seed, **(GROUND if ground else DYN))
    ast = env.global_tensor_dict["env_asset_state_tensor"]
    ast[..., 2] = torch.where(ast[..., 2] < -500.0, torch.full_like(ast[..., 2], 20.0), ast[..., 2])  # no parked assets
    env._repose_scene()
    return env


def test_no_contact_no_change():
    a, b = _high_env(True), _high_env(False)
    assert bool((a.global_tensor_dict["env_asset_state_tensor"][..., 2] > 9.0).all())
    g = torch.Generator(device=DEV).manual_seed(49)
    for step in range(15):
        act = (torch.rand(a.num_envs, a.num_robot_actions, generator=g, device=DEV) * 2 - 1) * 2.0
        tw = _twists(a, g)
        kw = {} if step % 5 == 4 else {"env_actions": tw}
        random.seed(700 + step)
        a.step(actions=act, **kw)
        random.seed(700 + step)
        b.step(actions=act, **kw)
        torch.cuda.synchronize()
        assert torch.equal(a.engine.root_state, b.engine.root_state), f"step {step}"
        for k in ("robot_contact_force_tensor", "env_asset_state_tensor"):
            assert torch.equal(a.global_tensor_dict[k], b.global_tensor_dict[k]), f"step {step}: {k}"
        assert torch.equal(a.collision_tensor, b.collision_tensor) and torch.equal(a._obj_pose, b._obj_pose)
    assert float(_lowest(a).min()) > 1.0


def test_graph_and_launch_modes_bit_identical_with_ground_contact():
    a = _env("dynamic_env", n=77, seed=50, step_mode="graph", **GROUND)
    b = _env("dynamic_env", n=77, seed=50, step_mode="launch", **GROUND)
    assert a.step_mode == "graph" and b.step_mode == "launch"
    g = torch.Generator(device=DEV).manual_seed(51)
    low0 = _lowest(a)
    for step in range(15):
        act = (torch.rand(a.num_envs, a.num_robot_actions, generator=g, device=DEV) * 2 - 1) * 3.0
        tw = _twists(a, g)
        kw = {} if step % 5 == 4 else {"env_actions": tw}
        random.seed(800 + step)
        a.step(actions=act, **kw)
        random.seed(800 + step)
        b.step(actions=act, **kw)
        torch.cuda.synchronize()
        assert torch.equal(a.engine.root_state, b.engine.root_state), f"step {step}"
        assert torch.equal(a.collision_tensor, b.collision_tensor)
        for k in ("robot_contact_force_tensor", "env_asset_state_tensor"):
            assert torch.equal(a.global_tensor_dict[k], b.global_tensor_dict[k]), f"step {step}: {k}"
        assert torch.equal(a._obj_pose, b._obj_pose) and torch.equal(a.scene.nodes, b.scene.nodes)
    active = (a.global_tensor_dict["env_asset_state_tensor"][..., 2] > -500.0).cpu().numpy()
    assert (low0[active] < -0.05).sum() > 20 and _lowest(a)[active].min() > low0[active].min()  # the ground solve ran
    assert {m for _, m in a._graphs} == {False, True}


def test_invalid_configurations_are_refused():
    for bad in ({**DYN, "contact_obstacle_ground": 1}, {"contact_moving_obstacles": True, "contact_obstacle_ground": True}):
        with pytest.raises(ValueError, match="contact_obstacle_ground"):
            _env("dynamic_env", n=4, **bad)
