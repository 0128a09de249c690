"""Rigid contact with dynamic obstacles (args['contact_dynamic_obstacles'], agx_hp2_contact_dynamic) on the GPU: the kernel against
the brute-force contact search + the numpy two-body solve of oracle/contact_dynamic_oracle.py in dynamic_env and among free trees;
bit identity with agx_hp2_contact_moving at infinite mass; a driven object that pushes a hovering robot less hard than a kinematic
one, a resting object knocked away by the robot, the velocity reset, graph and launch step modes bit-identical, and the refused
configurations."""
import random

import numpy as np
import pytest
import torch

from aerial_gym_simulator_b200 import _lib
from aerial_gym_simulator_b200.hp2 import ContactMotion, ObstacleMass, contact
from oracle import contact_dynamic_oracle as CD
from oracle import contact_oracle as CO
from tests.test_zz_contact_gpu import _env, _near_objects, object_tris
from tests.test_zz_contact_moving_gpu import _moving_test_env, _place, _twists, random_twists

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DYN = dict(contact_moving_obstacles=True, contact_dynamic_obstacles=True)


@pytest.fixture(autouse=True)
def _needs_the_kernels():
    if DEV == "cpu":  # the CPU dry run of the GPU test text: the contact kernels have no CPU twin
        pytest.skip("the contact kernels have no CPU twin")


def check_dynamic_against_oracle(scene, root, p, seed, asset_state, obj_asset, mass, max_ambiguous=0.25):
    """random robot velocities on the given poses and the given obstacle rows; kernel vs brute-force contacts + numpy two-body
    solve, with test_zz_contact_moving_gpu's tolerances and exclusion of ill-conditioned envs; the written asset rows too"""
    E = root.shape[0]
    g = torch.Generator().manual_seed(seed)
    root = root.clone()
    root[:, 7:13] = torch.randn(E, 6, generator=g) * 2.0
    got = root.to(DEV)
    st = asset_state.to(DEV).contiguous()
    force = torch.zeros(E, 3, device=DEV)
    crash = torch.zeros(E, dtype=torch.bool, device=DEV)
    ids = torch.zeros(E, _lib.CONTACT_MAX, dtype=torch.int32, device=DEV)
    contact(scene, got, p, force, crash, ids, motion=ContactMotion(st, obj_asset.to(DEV)), mass=ObstacleMass(mass.to(DEV)))
    torch.cuda.synchronize()
    cts, cnt, ref_ids, amb = CO.find_contacts(p, root[:, 0:3].numpy(), object_tris(scene), return_ambiguous=True)
    gid = ids.cpu().numpy()
    assert np.array_equal(np.sort(gid, axis=1), np.sort(ref_ids, axis=1)), "contact sets differ"
    for e in np.nonzero((gid != ref_ids).any(axis=1))[0]:  # ties to float32 rounding: take the kernel's order
        n = cnt[e]
        perm = [list(ref_ids[e, :n]).index(k) for k in gid[e, :n]]
        dist = p.radius - cts[e, :n, 6]
        moved = np.nonzero(np.arange(n) != np.asarray(perm))[0]
        assert np.ptp(dist[np.asarray(perm)[moved]]) <= 1e-5 * (1.0 + np.abs(dist).max()), f"env {e}: order {gid[e]} vs {ref_ids[e]}"
        cts[e, :n] = cts[e, perm]
    a0 = asset_state.numpy()
    ref, ref_f, ref_c, ref_st = CD.solve(p, root.numpy(), cts, cnt, gid, a0, obj_asset.numpy(), mass.numpy())
    g_, f_, s_ = got.cpu().numpy(), force.cpu().numpy(), st.cpu().numpy()
    assert np.array_equal(g_[:, 0:7], root[:, 0:7].numpy())
    assert amb.mean() < max_ambiguous
    ok = ~amb
    # rows the oracle leaves alone are bit-identical
    same = (ref_st == a0).all(axis=2)
    assert np.array_equal(s_[same], a0[same])
    tol = lambda a, b, s: np.abs(a - b) <= 5e-3 * (s + np.abs(b))
    vs = 1.0 + np.abs(a0[..., 7:13]).max(axis=(1, 2))[:, None] * 10.0
    bad = np.nonzero(ok & ~tol(g_[:, 7:13], ref[:, 7:13], vs).all(axis=1))[0]
    assert len(bad) == 0, f"max velocity error {np.abs(g_[ok, 7:13] - ref[ok, 7:13]).max()}: envs {bad[:8]}"
    assert tol(f_[ok], ref_f[ok], 10.0 * vs[ok]).all(), f"max force error {np.abs(f_[ok] - ref_f[ok]).max()}"
    assert tol(s_[ok][..., 7:13], ref_st[ok][..., 7:13], vs[ok][:, :, None]).all(), "asset twists differ"
    assert (np.abs(s_[ok][..., 0:7] - ref_st[ok][..., 0:7]) <= 1e-4 * (1.0 + np.abs(ref_st[ok][..., 0:7]))).all(), "asset poses differ"
    mag = np.linalg.norm(ref_f, axis=1)
    clear = ok & (np.abs(mag - p.force_threshold) > 1e-2 * (1.0 + p.force_threshold))
    assert np.array_equal(crash.cpu().numpy()[clear], ref_c[clear])
    assert (~same[ok]).any(), "no obstacle was pushed"
    return cnt


def test_dynamic_kernel_matches_oracle_in_dynamic_env():
    env = _env("dynamic_env", n=77, **DYN)
    p = env.contact_params
    st = random_twists(env.global_tensor_dict["env_asset_state_tensor"].cpu(), seed=23)
    mass = env._obstacle_mass.table.cpu()
    assert float(mass[..., 0].min()) > 0  # every dynamic_env object is a 1 kg body
    root = _near_objects(env.scene, env.num_envs, seed=8)
    cnt = check_dynamic_against_oracle(env.scene, root, p, 9, st, env._obj_asset.cpu(), mass)
    assert (cnt > 0).mean() > 0.3 and (cnt > 1).any()
    p.ground_plane = 1
    root[:, 2] = torch.rand(env.num_envs) * 0.4 - 0.05
    check_dynamic_against_oracle(env.scene, root, p, 10, st, env._obj_asset.cpu(), mass)


def _tree_env(n, seed):
    from aerial_gym_simulator_b200.config import asset_config as ac
    from aerial_gym_simulator_b200.config.env_config import DynamicEnvironmentCfg as base
    from aerial_gym_simulator_b200.registry._core import env_config_registry

    trees = type("contact_dynamic_trees", (ac.dynamic_tree_asset_params,), dict(num_assets=3, keep_in_env=False))

    class Cfg(base):
        class env_config(base.env_config):
            include_asset_type = {"trees": True}
            asset_type_to_dict_map = {"trees": trees}
    env_config_registry.register("contact_dynamic_tree_test_env", Cfg)
    return _env("contact_dynamic_tree_test_env", n=n, seed=seed, **DYN)


def test_dynamic_kernel_matches_oracle_among_free_trees():
    env = _tree_env(61, seed=24)
    p = env.contact_params
    mass = env._obstacle_mass.table.cpu()
    assert float(mass[..., 0].max()) < 1.0 / 12.0 and float(mass[..., 1:4].norm(dim=-1).min()) > 1.0  # 13 kg, COM off the base
    assert env.scene.K > env.num_obs_in_env  # multi-part assets
    st = random_twists(env.global_tensor_dict["env_asset_state_tensor"].cpu(), seed=25)
    root = _near_objects(env.scene, env.num_envs, seed=11, spread=0.4)
    cnt = check_dynamic_against_oracle(env.scene, root, p, 12, st, env._obj_asset.cpu(), mass, max_ambiguous=0.5)
    assert (cnt > 0).mean() > 0.3


def test_infinite_mass_is_bit_identical_to_the_moving_kernel():
    env = _env("dynamic_env", n=77, **DYN)
    p = env.contact_params
    st = random_twists(env.global_tensor_dict["env_asset_state_tensor"].cpu(), seed=26).to(DEV)
    root = _near_objects(env.scene, env.num_envs, seed=13).to(DEV)
    root[:, 7:13] = torch.randn(env.num_envs, 6, generator=torch.Generator().manual_seed(14)).to(DEV) * 2.0
    zero = ObstacleMass(torch.zeros(env.num_envs, env.num_obs_in_env, 13, device=DEV))
    out, rows = [], []
    for mass in (None, zero):
        rs, s = root.clone(), st.clone()
        f = torch.zeros(env.num_envs, 3, device=DEV)
        c = torch.zeros(env.num_envs, dtype=torch.bool, device=DEV)
        ids = torch.zeros(env.num_envs, _lib.CONTACT_MAX, dtype=torch.int32, device=DEV)
        contact(env.scene, rs, p, f, c, ids, motion=ContactMotion(s, env._obj_asset), mass=mass)
        out.append((rs, f, c, ids))
        rows.append(s)
    torch.cuda.synchronize()
    for a, b in zip(*out):
        assert torch.equal(a, b)
    assert torch.equal(rows[1], st) and bool((out[0][3][:, 0] >= 0).any())


def _peak_push(dynamic):
    args = dict(contact_dynamic_obstacles=True) if dynamic else {}
    env = _moving_test_env("contact_dynamic_push_test_env" + ("_d" if dynamic else "_m"), "objects", "1_x_1_wall.urdf", n=37,
                           seed=27, **args)
    R, u = env.robot.collision_radius, 2.0
    ast = env.global_tensor_dict["env_asset_state_tensor"]
    x0 = -(R + 0.05 + 0.3)
    _place(env, (0.0, 0.0, 2.0), (x0, 0.0, 2.0))
    twist = torch.zeros(env.num_envs, 2, 6, device=DEV)
    twist[:, 0, 0] = u
    act = torch.zeros(env.num_envs, env.num_robot_actions, device=DEV)
    peak = torch.zeros(env.num_envs, device=DEV)
    # one sub-step per env step, so that the force of every sub-step is seen (the tensor holds the last sub-step's)
    env.cfg.env.num_physics_steps_per_env_step_mean = 1
    for _ in range(80):
        env.reset_tensors()
        env.step(actions=act, env_actions=twist)
        peak = torch.maximum(peak, env.global_tensor_dict["robot_contact_force_tensor"].norm(dim=1))
    torch.cuda.synchronize()
    return peak, ast[:, 0, 0].clone(), env.engine.root_state[:, 0].clone()


def test_a_driven_object_pushes_a_hovering_robot_less_hard_than_a_kinematic_one():
    peak_m, box_m, rob_m = _peak_push(False)
    peak_d, box_d, rob_d = _peak_push(True)
    assert bool((peak_m > 0).all()) and bool((peak_d > 0).all())
    assert bool((peak_d < peak_m).all()), (float(peak_d.max()), float(peak_m.min()))
    assert bool((box_d < box_m - 1e-3).all())  # the pushed object lags its commanded path
    assert float(rob_d.min()) > 0.1  # and still pushes the robot away


def test_a_robot_knocks_a_resting_object_away():
    env = _moving_test_env("contact_dynamic_knock_test_env", "objects", "1_x_1_wall.urdf", n=37, seed=28, controller="no_control",
                           contact_dynamic_obstacles=True)
    R = env.robot.collision_radius
    ast = env.global_tensor_dict["env_asset_state_tensor"]
    bx = R + 0.05 + 0.05  # face 5 cm ahead of the sphere
    _place(env, (0.0, 0.0, 2.0), (bx, 0.0, 2.0))
    env.engine.root_state[:, 7] = 3.0
    act = torch.zeros(env.num_envs, env.num_robot_actions, device=DEV)
    env.step(actions=act)  # no env_actions: the object is a free body
    torch.cuda.synchronize()
    assert bool((ast[:, 0, 7] > 0.5).all()) and bool((ast[:, 0, 0] > bx + 0.03).all())
    assert float(ast[:, 0, 8:10].abs().max()) < 0.05
    assert bool((env.engine.root_state[:, 7] < 3.0).all())
    # the scene was re-posed after the last sub-step: the obstacle is where its row says, for the sensors and the next step
    assert torch.equal(env._obj_pose[:, 0], ast[:, 0, 0:7])
    probe = torch.zeros(env.num_envs, 13, device=DEV)
    probe[:, 0:3], probe[:, 6] = ast[:, 0, 0:3], 1.0
    probe[:, 0] -= 0.05  # on the object's near face (0.1 m thick) where it is now ...
    hit = torch.zeros(env.num_envs, dtype=torch.bool, device=DEV)
    env.scene.collide(probe, 0.01, hit)
    probe[:, 0] = bx - 0.05  # ... and where it was
    miss = torch.zeros_like(hit)
    env.scene.collide(probe, 0.01, miss)
    torch.cuda.synchronize()
    assert bool(hit.all()) and not bool(miss.any())
    # the next step without env_actions: it drifts on with its damped velocity
    x1, v1 = ast[:, 0, 0].clone(), ast[:, 0, 7].clone()
    env.engine.root_state[:, 0:3] = torch.tensor([-5.0, 0.0, 2.0], device=DEV)
    env.engine.root_state[:, 7:13] = 0.0
    env.step(actions=act)
    torch.cuda.synchronize()
    assert bool((ast[:, 0, 0] > x1 + 0.5 * v1 * 0.05).all()) and bool((ast[:, 0, 7] < v1).all())


def test_reset_zeroes_the_obstacle_velocities_of_the_reset_envs_only():
    env = _env("dynamic_env", n=45, seed=29, **DYN)
    ast = env.global_tensor_dict["env_asset_state_tensor"]
    ast[..., 7:13] = 1.5
    ids = torch.tensor([0, 3, 7, 44], device=DEV)
    env.reset_idx(ids)
    torch.cuda.synchronize()
    mask = torch.zeros(env.num_envs, dtype=torch.bool, device=DEV)
    mask[ids] = True
    assert bool((ast[mask][..., 7:13] == 0).all()) and bool((ast[~mask][..., 7:13] == 1.5).all())
    # without the key the reset writes positions and orientations only, as before
    ref = _env("dynamic_env", n=45, seed=29, contact_moving_obstacles=True)
    ra = ref.global_tensor_dict["env_asset_state_tensor"]
    ra[..., 7:13] = 1.5
    ref.reset_idx(ids)
    assert bool((ra[..., 7:13] == 1.5).all())


def test_graph_and_launch_modes_bit_identical_with_dynamic_obstacles():
    a = _env("dynamic_env", n=77, seed=30, step_mode="graph", **DYN)
    b = _env("dynamic_env", n=77, seed=30, step_mode="launch", **DYN)
    assert a.step_mode == "graph" and b.step_mode == "launch"
    g = torch.Generator(device=DEV).manual_seed(31)
    pushed = False
    for step in range(15):
        act = (torch.rand(a.num_envs, a.num_robot_actions, generator=g, device=DEV) * 2 - 1) * 3.0
        tw = _twists(a, g)
        kw = {} if step % 5 == 4 else {"env_actions": tw}  # some steps without env_actions: the obstacles drift
        random.seed(500 + step)
        a.step(actions=act, **kw)
        random.seed(500 + step)
        b.step(actions=act, **kw)
        torch.cuda.synchronize()
        assert torch.equal(a.engine.root_state, b.engine.root_state), f"step {step}"
        assert torch.equal(a.collision_tensor, b.collision_tensor)
        for k in ("robot_contact_force_tensor", "env_asset_state_tensor"):
            assert torch.equal(a.global_tensor_dict[k], b.global_tensor_dict[k]), f"step {step}: {k}"
        assert torch.equal(a._obj_pose, b._obj_pose) and torch.equal(a.scene.nodes, b.scene.nodes)
        pushed |= bool((a.global_tensor_dict["robot_contact_force_tensor"].norm(dim=1) > 0).any())
    assert pushed
    assert {m for _, m in a._graphs} == {False, True}


def test_invalid_configurations_are_refused():
    for bad in ({"contact_dynamic_obstacles": True}, {"contact_moving_obstacles": True, "contact_dynamic_obstacles": 1},
                {"contact_moving_obstacles": False, "contact_dynamic_obstacles": True}):
        with pytest.raises(ValueError, match="contact_dynamic_obstacles"):
            _env("dynamic_env", n=4, **bad)
    with pytest.raises(ValueError, match="contact_dynamic_obstacles"):  # a flag-mode env
        _env("dynamic_env", n=4, contact="flag", contact_dynamic_obstacles=True)
    with pytest.raises(ValueError, match="fix_base_link"):  # env_with_obstacles' assets are fixed
        _env("env_with_obstacles", n=4, **DYN)
    with pytest.raises(NotImplementedError):
        _env("empty_env", robot="base_quadrotor", controller="lee_velocity_control", n=8, host_io=True, **DYN)
