"""Rigid contact mode (args['contact'] = 'rigid', agx_hp2_contact) on the GPU: the kernel against the brute-force contact search
+ the numpy solve of oracle/contact_oracle.py in real envs, a mesh scene and a ground-only env; walls that hold; crashes on
ground contact; graph and launch step modes bit-identical."""
import random

import numpy as np
import pytest
import torch

from aerial_gym_simulator_b200 import _lib
from aerial_gym_simulator_b200.hp2 import RayScene, contact
from oracle import contact_oracle as CO
from oracle import hp2_oracle as RO
from tests import _hp2_mesh_common as HM

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(autouse=True)
def _needs_the_kernels():
    if DEV == "cpu":  # the CPU dry run of the GPU test text: the contact kernel has no CPU twin
        pytest.skip("the contact kernel has no CPU twin")


def _env(env_name, robot="lmf2", controller="lmf2_velocity_control", n=77, seed=3, **args):
    import aerial_gym_simulator_b200.task  # noqa: F401
    from aerial_gym_simulator_b200.sim import SimBuilder

    random.seed(seed)
    torch.manual_seed(seed)
    env = SimBuilder().build_env("base_sim", env_name, robot, controller, DEV, args={"seed": seed, "contact": "rigid", **args},
                                 num_envs=n, use_warp=True, headless=True)
    env.reset()
    return env


def object_tris(scene):
    """per env, per object: world triangles (a, ab, ac) with the oracle's transform arithmetic"""
    E, K = scene.E, scene.K
    cl, offs = scene.tmpl_tris.cpu().numpy().reshape(-1, 9), scene.tmpl_tri_offset.cpu().numpy()
    nT = int(scene.c.num_templates)
    tmesh = scene.tmpl_mesh.cpu().numpy() if scene.c.num_meshes else np.full(nT, -1)
    if scene.c.num_meshes:
        mt, mo = scene.mesh_tris.cpu().numpy().reshape(-1, 9), scene.mesh_tri_offset.cpu().numpy()
    allt = [mt[mo[m]:mo[m + 1]] if m >= 0 else cl[offs[t]:offs[t + 1]] for t, m in enumerate(tmesh)]
    o = np.concatenate([[0], np.cumsum([len(t) for t in allt])]).astype(np.int32)
    tt = np.concatenate(allt)
    pose = scene.obj_pose[..., :7].cpu().numpy().reshape(E * K, 1, 7)
    tm = scene.obj_template.cpu().numpy().reshape(E * K, 1)
    mx = max(len(t) for t in allt)
    tris, _, cnt = RO.build_world_tris(pose, tm, np.zeros_like(tm), o, tt, np.zeros(len(tt), np.int32), np.ones(len(tt), np.int32), mx)
    return [[tris[e * K + k, :cnt[e * K + k]] for k in range(K)] for e in range(E)]


def check_against_oracle(scene, root, p, seed):
    """random velocities on the given poses; kernel vs brute-force contacts + numpy solve"""
    E = root.shape[0]
    g = torch.Generator().manual_seed(seed)
    root = root.clone()
    root[:, 7:13] = torch.randn(E, 6, generator=g) * 2.0
    got = root.to(DEV)
    force = torch.zeros(E, 3, device=DEV)
    crash = torch.zeros(E, dtype=torch.bool, device=DEV)
    ids = torch.zeros(E, _lib.CONTACT_MAX, dtype=torch.int32, device=DEV)
    contact(scene, got, p, force, crash, ids)
    torch.cuda.synchronize()
    objs = object_tris(scene) if scene is not None else [[] for _ in range(E)]
    cts, cnt, ref_ids, amb = CO.find_contacts(p, root[:, 0:3].numpy(), objs, return_ambiguous=True)
    gid = ids.cpu().numpy()
    assert np.array_equal(np.sort(gid, axis=1), np.sort(ref_ids, axis=1)), "contact sets differ"
    for e in np.nonzero((gid != ref_ids).any(axis=1))[0]:
        # the same contacts in another order: only where their distances tie to float32 rounding; the solve then takes them in the
        # kernel's order
        n = cnt[e]
        perm = [list(ref_ids[e, :n]).index(k) for k in gid[e, :n]]
        dist = p.radius - cts[e, :n, 6]
        moved = np.nonzero(np.arange(n) != np.asarray(perm))[0]
        assert np.ptp(dist[np.asarray(perm)[moved]]) <= 1e-5 * (1.0 + np.abs(dist).max()), f"env {e}: order {gid[e]} vs {ref_ids[e]}"
        cts[e, :n] = cts[e, perm]
    ref, ref_f, ref_c = CO.solve(p, root.numpy(), cts, cnt)
    g_, f_ = got.cpu().numpy(), force.cpu().numpy()
    assert np.array_equal(g_[:, 0:7], root[:, 0:7].numpy())  # the pose is not projected
    # a centre on a medial plane of a solid has two closest points: the one float32 rounding picks differs, compare the rest
    assert amb.mean() < 0.25  # tessellated tree trunks have many near-equidistant faces around a centre inside them
    ok = ~amb
    # contact points and normals differ from the float64 search in the last float32 bits; a solve of up to 8 coupled contacts
    # that a few passes do not converge amplifies that, up to a few 1e-3 of the velocities
    tol = lambda a, b, s: np.abs(a - b) <= 5e-3 * (s + np.abs(b))
    err = np.abs(g_[ok, 7:13] - ref[ok, 7:13]).max()
    bad = np.nonzero(ok & ~tol(g_[:, 7:13], ref[:, 7:13], 1.0).all(axis=1))[0]
    assert len(bad) == 0, f"max velocity error {err}: envs {bad[:8]}, contacts {cnt[bad[:8]]}, depths {cts[bad[:2], :, 6]}"
    assert tol(f_[ok], ref_f[ok], 10.0).all(), f"max force error {np.abs(f_[ok] - ref_f[ok]).max()}"
    mag = np.linalg.norm(ref_f, axis=1)
    clear = ok & (np.abs(mag - p.force_threshold) > 1e-2 * (1.0 + p.force_threshold))
    assert np.array_equal(crash.cpu().numpy()[clear], ref_c[clear])
    return cnt


def _near_objects(scene, E, seed, spread=0.8):
    """robot centres scattered around a random object of each env, so that most envs touch something"""
    g = torch.Generator().manual_seed(seed)
    pose = scene.obj_pose[..., 0:3].cpu()
    k = torch.randint(0, scene.K, (E,), generator=g)
    root = torch.zeros(E, 13)
    root[:, 0:3] = pose[torch.arange(E), k] + (torch.rand(E, 3, generator=g) * 2 - 1) * spread
    q = torch.randn(E, 4, generator=g)
    root[:, 3:7] = q / q.norm(dim=1, keepdim=True)
    return root


@pytest.mark.parametrize("env_name", ["env_with_obstacles", "forest_env"])
def test_kernel_matches_oracle_in_envs(env_name):
    env = _env(env_name, n=77)
    p = env.contact_params
    root = _near_objects(env.scene, env.num_envs, seed=1)
    cnt = check_against_oracle(env.scene, root, p, seed=2)
    assert (cnt > 0).mean() > 0.3 and (cnt > 1).any()
    p.ground_plane = 1  # the same scene with a floor
    root[:, 2] = torch.rand(env.num_envs) * 0.4 - 0.05
    check_against_oracle(env.scene, root, p, seed=3)


def test_kernel_matches_oracle_in_a_mesh_scene():
    E = 45
    sc = HM.make_mixed_scene(E, 10, seed=21, extent=2.0, parked=2)
    t, b, m = HM.scene_templates(sc)
    scene = RayScene(t, b, m, sc["tm"], sc["ctr"], sc["pose"].to(DEV), DEV, mesh_templates=sc["meshes"])
    scene.update()
    p = _lib.AgxContactParams(radius=0.25, contact_offset=0.01, rest_offset=0.005, dt=0.01, mass=0.9, friction=0.7,
                              max_depenetration_velocity=1.0, force_threshold=5.0, iterations=6, ground_plane=0)
    p.inertia_inv[:] = [60.0, 0, 0, 0, 55.0, 0, 0, 0, 30.0]
    p.com[:] = [0.0, 0.0, 0.01]
    cnt = check_against_oracle(scene, _near_objects(scene, E, seed=4, spread=1.0), p, seed=5)
    assert (cnt > 0).mean() > 0.3


def test_kernel_matches_oracle_ground_only():
    env = _env("empty_env", n=100)
    p = env.contact_params
    p.ground_plane = 1
    assert env.scene is None
    g = torch.Generator().manual_seed(6)
    root = torch.zeros(env.num_envs, 13)
    root[:, 0:2] = torch.rand(env.num_envs, 2, generator=g)
    root[:, 2] = (torch.rand(env.num_envs, generator=g) * 2.5 - 0.5) * p.radius
    root[:, 6] = 1.0
    cnt = check_against_oracle(None, root, p, seed=7)
    assert 0 < (cnt > 0).sum() < env.num_envs


def test_walls_hold_without_reset_on_collision():
    from aerial_gym_simulator_b200.config.env_config import EnvWithObstaclesCfg as base
    from aerial_gym_simulator_b200.registry._core import env_config_registry

    class Cfg(base):
        class env(base.env):
            reset_on_collision = False
    env_config_registry.register("contact_walls_test_env", Cfg)
    env = _env("contact_walls_test_env", n=200, seed=8)
    assert not env.cfg.env.reset_on_collision
    g = torch.Generator(device=DEV).manual_seed(9)
    worst = 0.0
    for step in range(1000):
        act = (torch.rand(env.num_envs, env.num_robot_actions, generator=g, device=DEV) * 2 - 1) * 3.0
        env.step(actions=act)
        env.reset_terminated_and_truncated_envs()
        pos, lo, hi = env.engine.root_state[:, 0:3], env.engine.bounds_min, env.engine.bounds_max
        worst = max(worst, float(torch.maximum(lo - pos, pos - hi).max()))
    assert worst <= 0.02, f"a robot centre left its env bounds by {worst:.3f} m"
    assert env.global_tensor_dict["robot_contact_force_tensor"].abs().sum() > 0


def test_dynamic_env_flags_ground_contact():
    env = _env("dynamic_env", n=64, seed=10)
    assert env.contact_params.ground_plane == 1
    rs = env.engine.root_state
    rs[:, 2] = env.robot.collision_radius * 0.5  # half the sphere below z = 0
    rs[:, 7:13] = 0.0
    env.reset_tensors()
    env.step(actions=torch.zeros(env.num_envs, env.num_robot_actions, device=DEV))
    torch.cuda.synchronize()
    assert bool(env.collision_tensor.all())
    # the force is the last sub-step's: by then the floor has pushed some robots clear of it
    f = env.global_tensor_dict["robot_contact_force_tensor"]
    assert float(f[:, 2].max()) > env.cfg.env.collision_force_threshold


def test_graph_and_launch_modes_bit_identical():
    a, b = _env("env_with_obstacles", n=77, seed=11, step_mode="graph"), _env("env_with_obstacles", n=77, seed=11, step_mode="launch")
    assert a.step_mode == "graph" and b.step_mode == "launch"
    g = torch.Generator(device=DEV).manual_seed(12)
    for step in range(15):
        act = (torch.rand(a.num_envs, a.num_robot_actions, generator=g, device=DEV) * 2 - 1) * 3.0
        random.seed(200 + step)
        a.step(actions=act)
        random.seed(200 + step)
        b.step(actions=act)
        torch.cuda.synchronize()
        assert torch.equal(a.engine.root_state, b.engine.root_state), f"step {step}"
        assert torch.equal(a.collision_tensor, b.collision_tensor)
        fa, fb = (e.global_tensor_dict["robot_contact_force_tensor"] for e in (a, b))
        assert torch.equal(fa, fb)
    assert len(a._graphs) >= 1


def test_host_io_is_refused():
    with pytest.raises(NotImplementedError):
        _env("empty_env", robot="base_quadrotor", controller="lee_velocity_control", n=8, host_io=True)
