"""Rigid contact with moving obstacles (args['contact_moving_obstacles'], agx_hp2_contact_moving) on the GPU: the kernel against the
brute-force contact search + the numpy moving solve of oracle/contact_moving_oracle.py with random obstacle twists; its reduction to
agx_hp2_contact at zero twist; a moving box that pushes a hovering robot and a moving platform that carries one; obstacle states and
scenes bit-identical to the default order; graph and launch step modes bit-identical."""
import random

import numpy as np
import pytest
import torch

from aerial_gym_simulator_b200 import _lib
from aerial_gym_simulator_b200.hp2 import ContactMotion, RayScene, contact
from oracle import contact_moving_oracle as CM
from oracle import contact_oracle as CO
from tests import _hp2_mesh_common as HM
from tests.test_zz_contact_gpu import _env, _near_objects, object_tris

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(autouse=True)
def _needs_the_kernels():
    if DEV == "cpu":  # the CPU dry run of the GPU test text: the contact kernels have no CPU twin
        pytest.skip("the contact kernels have no CPU twin")


def random_twists(asset_state, seed):
    """asset rows with random velocities (|v| <= 3 m/s, |w| <= 2 rad/s), poses untouched"""
    st = asset_state.clone()
    g = torch.Generator().manual_seed(seed)
    E, A = st.shape[:2]
    d = torch.randn(E, A, 6, generator=g)
    st[..., 7:10] = d[..., 0:3] / d[..., 0:3].norm(dim=-1, keepdim=True) * torch.rand(E, A, 1, generator=g) * 3.0
    st[..., 10:13] = d[..., 3:6] / d[..., 3:6].norm(dim=-1, keepdim=True) * torch.rand(E, A, 1, generator=g) * 2.0
    return st


def check_moving_against_oracle(scene, root, p, seed, asset_state, obj_asset):
    """random robot velocities on the given poses, the given obstacle rows; kernel vs brute-force contacts + numpy moving solve, with
    the tolerances and the exclusion of ill-conditioned envs of test_zz_contact_gpu.check_against_oracle.  Its velocity scale 1.0 (the
    robot's random velocities) becomes 1 + the env's largest obstacle point speed: a 20 m wall turning at 2 rad/s moves its far
    corners at 20 m/s, and the rounding of a contact point or normal perturbs the solve in proportion to the relative velocity."""
    E = root.shape[0]
    g = torch.Generator().manual_seed(seed)
    root = root.clone()
    root[:, 7:13] = torch.randn(E, 6, generator=g) * 2.0
    got = root.to(DEV)
    force = torch.zeros(E, 3, device=DEV)
    crash = torch.zeros(E, dtype=torch.bool, device=DEV)
    ids = torch.zeros(E, _lib.CONTACT_MAX, dtype=torch.int32, device=DEV)
    contact(scene, got, p, force, crash, ids, motion=ContactMotion(asset_state.to(DEV), obj_asset.to(DEV)))
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
    u = CM.obstacle_point_velocity(asset_state.numpy(), obj_asset.numpy(), cts, gid)
    ref, ref_f, ref_c = CM.solve(p, root.numpy(), cts, cnt, obstacle_velocity=u)
    g_, f_ = got.cpu().numpy(), force.cpu().numpy()
    assert np.array_equal(g_[:, 0:7], root[:, 0:7].numpy())
    assert amb.mean() < 0.25
    ok = ~amb
    tol = lambda a, b, s: np.abs(a - b) <= 5e-3 * (s + np.abs(b))
    vs = 1.0 + np.linalg.norm(u, axis=2).max(axis=1, keepdims=True)
    bad = np.nonzero(ok & ~tol(g_[:, 7:13], ref[:, 7:13], vs).all(axis=1))[0]
    assert len(bad) == 0, f"max velocity error {np.abs(g_[ok, 7:13] - ref[ok, 7:13]).max()}: envs {bad[:8]}, scale {vs[bad[:8], 0]}"
    assert tol(f_[ok], ref_f[ok], 10.0 * vs[ok]).all(), f"max force error {np.abs(f_[ok] - ref_f[ok]).max()}"
    mag = np.linalg.norm(ref_f, axis=1)
    clear = ok & (np.abs(mag - p.force_threshold) > 1e-2 * (1.0 + p.force_threshold))
    assert np.array_equal(crash.cpu().numpy()[clear], ref_c[clear])
    # the obstacle velocities do change the outcome
    static, _, _ = CO.solve(p, root.numpy(), cts, cnt)
    assert not np.array_equal(ref[ok, 7:13], static[ok, 7:13])
    return cnt


@pytest.mark.parametrize("env_name", ["dynamic_env", "env_with_obstacles"])
def test_moving_kernel_matches_oracle_in_envs(env_name):
    env = _env(env_name, n=77, contact_moving_obstacles=True)
    p = env.contact_params
    st = random_twists(env.global_tensor_dict["env_asset_state_tensor"].cpu(), seed=13)
    root = _near_objects(env.scene, env.num_envs, seed=1)
    cnt = check_moving_against_oracle(env.scene, root, p, 2, st, env._obj_asset.cpu())
    assert (cnt > 0).mean() > 0.3 and (cnt > 1).any()
    p.ground_plane = 1
    root[:, 2] = torch.rand(env.num_envs) * 0.4 - 0.05
    check_moving_against_oracle(env.scene, root, p, 3, st, env._obj_asset.cpu())


def _mesh_scene(E):
    sc = HM.make_mixed_scene(E, 10, seed=21, extent=2.0, parked=2)
    t, b, m = HM.scene_templates(sc)
    scene = RayScene(t, b, m, sc["tm"], sc["ctr"], sc["pose"].to(DEV), DEV, mesh_templates=sc["meshes"])
    scene.update()
    p = _lib.AgxContactParams(radius=0.25, contact_offset=0.01, rest_offset=0.005, dt=0.01, mass=0.9, friction=0.7,
                              max_depenetration_velocity=1.0, force_threshold=5.0, iterations=6, ground_plane=0)
    p.inertia_inv[:] = [60.0, 0, 0, 0, 55.0, 0, 0, 0, 30.0]
    p.com[:] = [0.0, 0.0, 0.01]
    return sc, scene, p


def test_moving_kernel_matches_oracle_in_a_mesh_scene():
    E = 45
    sc, scene, p = _mesh_scene(E)
    # each object its own asset, its row = its pose
    st = torch.zeros(E, scene.K, 13)
    st[..., 0:7] = sc["pose"][..., 0:7]
    st = random_twists(st, seed=14)
    obj_asset = torch.arange(scene.K, dtype=torch.int32).expand(E, -1).contiguous()
    cnt = check_moving_against_oracle(scene, _near_objects(scene, E, seed=4, spread=1.0), p, 5, st, obj_asset)
    assert (cnt > 0).mean() > 0.3


def test_zero_twist_is_bit_identical_to_the_static_kernel():
    env = _env("dynamic_env", n=77, contact_moving_obstacles=True)
    p = env.contact_params
    st = env.global_tensor_dict["env_asset_state_tensor"].clone()
    st[..., 7:13] = 0.0
    root = _near_objects(env.scene, env.num_envs, seed=6).to(DEV)
    root[:, 7:13] = torch.randn(env.num_envs, 6, generator=torch.Generator().manual_seed(7)).to(DEV) * 2.0
    out = []
    for motion in (None, ContactMotion(st, env._obj_asset)):
        rs = root.clone()
        f = torch.zeros(env.num_envs, 3, device=DEV)
        c = torch.zeros(env.num_envs, dtype=torch.bool, device=DEV)
        ids = torch.zeros(env.num_envs, _lib.CONTACT_MAX, dtype=torch.int32, device=DEV)
        contact(env.scene, rs, p, f, c, ids, motion=motion)
        out.append((rs, f, c, ids))
    torch.cuda.synchronize()
    for a, b in zip(*out):
        assert torch.equal(a, b)
    assert bool((out[0][3][:, 0] >= 0).any()) and bool(out[0][2].any())


def _moving_test_env(name, folder, file, n, seed, controller="lmf2_velocity_control", **args):
    """dynamic_env with two copies of one asset file, reset_on_collision = False; the second copy is parked far away"""
    from aerial_gym_simulator_b200.config import asset_config as ac
    from aerial_gym_simulator_b200.config.env_config import DynamicEnvironmentCfg as base
    from aerial_gym_simulator_b200.registry._core import env_config_registry

    obj = type(name + "_objects", (ac.dynamic_object_asset_params,),
               dict(num_assets=2, asset_folder=f"{ac._ENV_ASSETS}/{folder}", file=file, keep_in_env=False))

    class Cfg(base):
        class env(base.env):
            reset_on_collision = False

        class env_config(base.env_config):
            include_asset_type = {"objects": True}
            asset_type_to_dict_map = {"objects": obj}
    env_config_registry.register(name, Cfg)
    env = _env(name, controller=controller, n=n, seed=seed, contact_moving_obstacles=True, **args)
    ast = env.global_tensor_dict["env_asset_state_tensor"]
    ast.zero_()
    ast[..., 6] = 1.0
    ast[:, 1, 0:3] = -1000.0
    return env


def _place(env, robot_pos, box_pos):
    rs, ast = env.engine.root_state, env.global_tensor_dict["env_asset_state_tensor"]
    rs[:, 0:3] = torch.tensor(robot_pos, device=DEV)
    rs[:, 3:7] = torch.tensor([0.0, 0.0, 0.0, 1.0], device=DEV)
    rs[:, 7:13] = 0.0
    ast[:, 0, 0:3] = torch.tensor(box_pos, device=DEV)
    env._repose_scene()
    env.reset_tensors()


def test_a_moving_box_pushes_a_hovering_robot():
    env = _moving_test_env("contact_moving_push_test_env", "objects", "1_x_1_wall.urdf", n=37, seed=15)  # box 0.1 x 1 x 1
    p, R, u = env.contact_params, env.robot.collision_radius, 2.0
    ast = env.global_tensor_dict["env_asset_state_tensor"]
    _place(env, (0.0, 0.0, 2.0), (-(R + 0.05 + 0.3), 0.0, 2.0))  # face 0.3 m from the sphere
    twist = torch.zeros(env.num_envs, 2, 6, device=DEV)
    twist[:, 0, 0] = u
    act = torch.zeros(env.num_envs, env.num_robot_actions, device=DEV)
    md = torch.zeros(env.num_envs, device=DEV)
    dummy = torch.zeros(env.num_envs, dtype=torch.bool, device=DEV)
    crashed, touched, worst = torch.zeros_like(dummy), torch.zeros_like(dummy), -1.0
    for step in range(8):
        env.reset_tensors()
        env.step(actions=act, env_actions=twist)
        crashed |= env.collision_tensor
        f = env.global_tensor_dict["robot_contact_force_tensor"]
        now = f.norm(dim=1) > 0
        touched |= now
        v, vbox = env.engine.root_state[:, 7], ast[:, 0, 7]  # the box moves at the damped twist, 2 m/s (1 - dt linear_damping)
        assert bool((v[now] >= vbox[now] * (1 - 1e-5)).all()), f"step {step}: robot slower than the box: {float(v[now].min())}"
        env.scene.collide(env.engine.root_state, R, dummy, md)
        worst = max(worst, float((R - md).max()))
    bound = p.rest_offset + u * p.dt + 9.81 * p.dt ** 2
    # the impact flags every robot; afterwards the solve's separating velocity lets the robot run slightly ahead and the box
    # catches up again, so not every env is in contact at the end of every env step
    assert bool(crashed.all()) and bool(touched.any())
    assert worst <= bound + 1e-4, f"penetration {worst:.4f} m > {bound:.4f} m"
    assert float(env.engine.root_state[:, 0].min()) > 0.3  # pushed well away from where it hovered


def test_a_moving_platform_carries_a_resting_robot():
    env = _moving_test_env("contact_moving_carry_test_env", "walls", "bottom_wall.urdf", n=37, seed=16,
                           controller="no_control")  # 20 x 20 x 0.2 plate
    R, u = env.robot.collision_radius, 1.0
    _place(env, (0.0, 0.0, 1.0 + R + 0.02), (0.0, 0.0, 1.0 - 0.1))  # top face z = 1, the robot 2 cm above it
    twist = torch.zeros(env.num_envs, 2, 6, device=DEV)
    twist[:, 0, 1] = u  # sideways, +y
    act = torch.zeros(env.num_envs, env.num_robot_actions, device=DEV)
    for step in range(15):
        env.step(actions=act, env_actions=twist)
    torch.cuda.synchronize()
    rs, ast = env.engine.root_state, env.global_tensor_dict["env_asset_state_tensor"]
    assert float(rs[:, 2].min()) > 1.0 + R - 0.02 and float(rs[:, 2].max()) < 1.0 + R + 0.02  # resting on the plate
    assert bool((env.global_tensor_dict["robot_contact_force_tensor"][:, 2] > 0).all())
    # friction carries it: its velocity at the contact point (below the centre, on the top face) is the plate's.  (A sphere whose
    # inertia is small against m R^2 mostly spins rather than translates when a belt moves under it.)
    x, y, z, w = rs[:, 3], rs[:, 4], rs[:, 5], rs[:, 6]
    Rm = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                      2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                      2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], dim=1).view(-1, 3, 3)
    com = rs[:, 0:3] + Rm @ torch.tensor(list(env.contact_params.com), device=DEV)
    p = rs[:, 0:3].clone()
    p[:, 2] = 1.0
    vp = rs[:, 7:10] + torch.cross(rs[:, 10:13], p - com, dim=1)
    # tangential part only: normally the solve leaves the at-rest separating velocity g dt (DESIGN "At rest")
    assert float((vp[:, 0:2] - ast[:, 0, 7:9]).abs().max()) < 0.02 * u, vp
    assert float(ast[0, 0, 8]) > 0.99 * u


def _twists(env, g, scale=2.0):
    return (torch.rand(env.num_envs, env.num_obs_in_env, 6, generator=g, device=DEV) * 2 - 1) * scale


def test_obstacles_and_scene_bit_identical_to_the_default_order():
    a = _env("dynamic_env", n=45, seed=17)
    b = _env("dynamic_env", n=45, seed=17, contact_moving_obstacles=True)
    g = torch.Generator(device=DEV).manual_seed(18)
    for step in range(6):
        act = (torch.rand(a.num_envs, a.num_robot_actions, generator=g, device=DEV) * 2 - 1) * 3.0
        tw = _twists(a, g)
        random.seed(300 + step)
        a.step(actions=act, env_actions=tw)
        random.seed(300 + step)
        b.step(actions=act, env_actions=tw)
        torch.cuda.synchronize()
        sa, sb = (e.global_tensor_dict["env_asset_state_tensor"] for e in (a, b))
        assert torch.equal(sa, sb), f"step {step}"
        for name in ("tris", "nodes", "leaf_object", "obb"):
            assert torch.equal(getattr(a.scene, name), getattr(b.scene, name)), f"step {step}: scene {name}"
    assert len(b._graphs) >= 1 and all(k[1] for k in b._graphs)


def test_graph_and_launch_modes_bit_identical_with_moving_obstacles():
    a = _env("dynamic_env", n=77, seed=19, step_mode="graph", contact_moving_obstacles=True)
    b = _env("dynamic_env", n=77, seed=19, step_mode="launch", contact_moving_obstacles=True)
    assert a.step_mode == "graph" and b.step_mode == "launch"
    g = torch.Generator(device=DEV).manual_seed(20)
    for step in range(15):
        act = (torch.rand(a.num_envs, a.num_robot_actions, generator=g, device=DEV) * 2 - 1) * 3.0
        tw = _twists(a, g)
        kw = {} if step % 5 == 4 else {"env_actions": tw}  # some steps without env_actions: the static graph
        random.seed(400 + step)
        a.step(actions=act, **kw)
        random.seed(400 + step)
        b.step(actions=act, **kw)
        torch.cuda.synchronize()
        assert torch.equal(a.engine.root_state, b.engine.root_state), f"step {step}"
        assert torch.equal(a.collision_tensor, b.collision_tensor)
        for k in ("robot_contact_force_tensor", "env_asset_state_tensor"):
            assert torch.equal(a.global_tensor_dict[k], b.global_tensor_dict[k]), f"step {step}: {k}"
    assert {m for _, m in a._graphs} == {False, True}


def test_host_io_is_refused():
    with pytest.raises(NotImplementedError):
        _env("empty_env", robot="base_quadrotor", controller="lee_velocity_control", n=8, host_io=True, contact_moving_obstacles=True)
