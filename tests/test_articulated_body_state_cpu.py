"""Per-body state of articulated robots on the CPU (DESIGN.md "Articulated robots"): art_body_states of articulated_core.cuh (host
shadow, tests/csrc/articulated_shadow.cu) against oracle/articulated_body_state_oracle.py's float64 body_states(), the Global Tensor
Dict keys and their refresh in EnvManager, ray-cast sensors on a link (cfg.parent_link), and the gimbal quadrotor's levelling."""
import numpy as np
import pytest
import torch

from oracle import articulated_body_state_oracle as BO
from oracle import articulated_oracle as AO
from oracle import hp2_oracle as RO

from . import _articulated_shadow
from . import _hp2_common as H2
from ._cpu_stack_articulated import articulated_cpu_stack
from .test_articulated_cpu import morphy_compliant, random_art, random_root, table_of

EPS = float(np.finfo(np.float32).eps)


def _path(table, i):
    """the bodies from i up to (not including) the root"""
    out = []
    while i > 0:
        out.append(i)
        i = int(table["parent"][i])
    return out


def _shadow_rows(art_spec, roots, dof):
    """roots [N,13], dof [N,D,2] -> shadow rows [N,B,13] (float32)"""
    s = art_spec.to_struct()
    dof_t = torch.tensor(np.asarray(dof, np.float32)).contiguous()
    s.dof_state = dof_t.data_ptr()
    root_t = torch.tensor(np.asarray(roots, np.float32))
    out = torch.zeros(root_t.shape[0], s.num_bodies, 13)
    _articulated_shadow.body_state(s, root_t, out)
    return out.numpy(), s, root_t.numpy()


def _check_rows(table, root, dof, rows):
    """Tolerance, per body i of depth d (joints between it and the root), path length L = sum |joint_p| along the path and joint
    speed Q = sum |q-dot| along the path.  Each level rounds a quaternion -> matrix, two 3x3 products, the axis-angle matrix (sincosf is
    within 2 ulp for any float argument, so |q| of 200 rad costs nothing) and the matrix -> quaternion conversion: about 20 float32 ulps
    of a unit rotation, so the rotation may be off by e_R = 32 eps (d + 1) (compared as matrices: the quaternion's sign is free).  A
    rotation error moves the lever arms: the position gets e_R L on top of one rounding of the world position (2 eps |x0|, what a root
    1000 m out costs) and 8 eps L; the angular velocity gets e_R Q + 8 eps (|w0| + Q); the linear velocity e_R Q L (twice: P x a and
    w x P) + e_w L + 8 eps (|v0| + (|w| + Q) L)."""
    ref = BO.body_states(table, root, dof[:, 0], dof[:, 1])
    assert np.array_equal(rows[0], np.asarray(root, np.float32)), "row 0 is the root row, bit for bit"
    worst = 0.0
    for i in range(1, int(table["num_bodies"])):
        p = _path(table, i)
        d, L, Q = len(p), sum(float(np.linalg.norm(table["joint_p"][k])) for k in p), sum(abs(float(dof[k - 1, 1])) for k in p)
        eR = 32 * EPS * (d + 1)
        tol_x = 2 * EPS * np.abs(root[0:3]).max() + eR * L + 8 * EPS * L
        tol_w = eR * Q + 8 * EPS * (np.linalg.norm(root[10:13]) + Q)
        wn = np.linalg.norm(ref[i, 10:13])
        tol_v = 2 * eR * Q * L + tol_w * L + 8 * EPS * (np.linalg.norm(root[7:10]) + (wn + Q) * L)
        Rg, Rr = AO.quat_to_matrix(rows[i, 3:7]), AO.quat_to_matrix(ref[i, 3:7])
        for err, tol in ((np.abs(Rg - Rr).max(), eR), (np.abs(rows[i, 0:3] - ref[i, 0:3]).max(), tol_x),
                         (np.abs(rows[i, 10:13] - ref[i, 10:13]).max(), tol_w), (np.abs(rows[i, 7:10] - ref[i, 7:10]).max(), tol_v)):
            assert err <= tol, (i, err, tol)
            worst = max(worst, err / tol)
        assert abs(np.linalg.norm(rows[i, 3:7]) - 1.0) < 8 * EPS
    return worst


def _cases(rng, B, n):
    roots, dofs = [], []
    for k in range(n):
        r = random_root(rng)
        if k % 2:
            r[0:3] = rng.uniform(-1000, 1000, 3)  # far from the origin
        q = rng.uniform(-3, 3, B - 1)
        if k % 3 == 0:
            q = rng.choice([-1, 1], B - 1) * rng.uniform(40, 200, B - 1)  # continuous joints, many turns
        roots.append(r)
        dofs.append(np.stack([q, rng.uniform(-3, 3, B - 1)], -1) if B > 1 else np.zeros((0, 2)))
    return np.array(roots, np.float32), np.array(dofs, np.float32).reshape(n, B - 1, 2)


def test_shadow_matches_oracle_on_morphy_compliant():
    _, art = morphy_compliant()
    roots, dofs = _cases(np.random.default_rng(0), art.bodies.num_bodies, 64)
    rows, s, roots32 = _shadow_rows(art, roots, dofs)
    table = table_of(s)
    for n in range(len(roots)):
        _check_rows(table, roots32[n].astype(np.float64), dofs[n].astype(np.float64), rows[n])


@pytest.mark.parametrize("B", [1, 2, 3, 9, 10, 16])
def test_shadow_matches_oracle_on_random_trees(B):
    rng = np.random.default_rng(B)
    worst = 0.0
    for t in range(4):
        art = random_art(rng, B)
        roots, dofs = _cases(rng, B, 16)
        rows, s, roots32 = _shadow_rows(art, roots, dofs)
        table = table_of(s)
        for n in range(len(roots)):
            worst = max(worst, _check_rows(table, roots32[n].astype(np.float64), dofs[n].astype(np.float64), rows[n]))
    assert worst <= 1.0


def _fk(table, root, q):
    R, P, _ = AO.kinematics(table, root[3:7], q)
    return R, P + root[0:3]


def test_velocities_are_the_time_derivatives_of_the_forward_kinematics():
    """central differences of the float64 FK along x0 + v t, exp(w t) R0, q + q-dot t"""
    rng = np.random.default_rng(5)
    h = 1e-6
    for B in (2, 9, 16):
        art = random_art(rng, B)
        table = table_of(art.to_struct())
        root = random_root(rng)
        q, qd = rng.uniform(-2, 2, B - 1), rng.uniform(-2, 2, B - 1)
        ref = BO.body_states(table, root, q, qd)
        w = root[10:13]

        def at(t):
            r = root.copy()
            r[0:3] = root[0:3] + root[7:10] * t
            Rw = AO._rot(w / np.linalg.norm(w), np.linalg.norm(w) * t) @ AO.quat_to_matrix(root[3:7])
            r[3:7] = BO.matrix_to_quat(Rw)
            return _fk(table, r, q + qd * t)
        (Rp, Pp), (Rm, Pm) = at(h), at(-h)
        R0, _ = at(0.0)
        for i in range(B):
            assert np.abs((Pp[i] - Pm[i]) / (2 * h) - ref[i, 7:10]).max() < 1e-6
            W = (Rp[i] - Rm[i]) / (2 * h) @ R0[i].T
            assert np.abs(np.array([W[2, 1], W[0, 2], W[1, 0]]) - ref[i, 10:13]).max() < 1e-6


# ---- EnvManager ---------------------------------------------------------------------------------------------------------------
def _env(robot="morphy_compliant", env_name="empty_env", n=8, **args):
    from aerial_gym_simulator_b200.env_manager.env_manager import EnvManager
    return EnvManager("base_sim", env_name, robot, "lee_attitude_control", "cpu", num_envs=n, args=args or None)


def _expected_rows(env):
    eng = env.engine
    out = torch.zeros_like(eng.body_state)
    _articulated_shadow.body_state(eng.art, eng.root_state, out)
    return out


def test_gtd_keys_and_refresh_after_step_and_reset():
    with articulated_cpu_stack():
        torch.manual_seed(0)
        env = _env(n=8)
        gtd = env.global_tensor_dict
        bs = gtd["robot_body_state_tensor"]
        assert bs.shape == (8, 9, 13) and bs is env.engine.body_state
        assert gtd["robot_body_names"] == list(env.robot.bodies.links) and gtd["robot_body_names"][0] == "base_link"
        env.reset()
        assert torch.equal(bs, _expected_rows(env))
        gtd["dof_position_setpoint_tensor"].fill_(0.2)
        for _ in range(3):
            env.step(torch.rand(8, 4) * 0.2)
            assert torch.equal(bs, _expected_rows(env))
            assert torch.equal(bs[:, 0], gtd["robot_state_tensor"])
        env.simulate(torch.zeros(8, 4))
        assert torch.equal(bs, _expected_rows(env))
        before = bs.clone()
        env.reset_idx(torch.tensor([1, 5]))
        assert torch.equal(bs, _expected_rows(env))
        changed = (bs != before).flatten(1).any(1)
        assert changed[[1, 5]].all() and not changed[[0, 2, 3, 4, 6, 7]].any()
        state = torch.get_rng_state()
        env.engine.update_body_state()
        assert torch.equal(torch.get_rng_state(), state)


def test_rigid_robots_get_no_body_keys():
    with articulated_cpu_stack():
        env = _env("base_quadrotor", n=4)
        assert "robot_body_state_tensor" not in env.global_tensor_dict and "robot_body_names" not in env.global_tensor_dict
        assert env.engine.body_state is None
        with pytest.raises(ValueError):
            env.engine.update_body_state()


# ---- sensors on a link ----------------------------------------------------------------------------------------------------------
def _oracle_image(env, pose, mount, idx=None):
    sc = env.scene
    tris, segs, cnt = RO.build_world_tris(env._obj_pose.cpu().numpy(), sc.obj_template.cpu().numpy(), sc.obj_seg_counter.cpu().numpy(),
                                          sc.tmpl_tri_offset.cpu().numpy(), sc.tmpl_tris.cpu().numpy(), sc.tmpl_seg_base.cpu().numpy(),
                                          sc.tmpl_seg_mask.cpu().numpy(), sc.K * sc.L)
    idx = np.arange(len(pose)) if idx is None else idx
    so, _ = H2.oracle_sensor(env.sensor_cfg)
    return RO.cast(so, np.ascontiguousarray(pose[idx]), np.ascontiguousarray(mount[idx]), None, tris[idx], segs[idx], cnt[idx])


def gimbal_camera_check(env, idx=None):
    """the image equals the brute-force oracle's at the pose built from the published row of the camera link's body, T_l and the
    mount -- bit for bit"""
    gtd = env.global_tensor_dict
    b = gtd["robot_body_names"].index("pitch_stage_link")
    R_l, p_l = env.robot.bodies.link_in_body["gimbal_camera_link"]
    assert env.robot.bodies.link_body["gimbal_camera_link"] == b and np.array_equal(R_l, np.eye(3))
    pose = gtd["robot_body_state_tensor"][:, b, :7].cpu().numpy()
    mount = env.sensor_mount.cpu().numpy().copy()
    mount[..., 0:3] = mount[..., 0:3] + np.asarray(p_l, np.float32)  # T_l = (1, p_l): folded by hand
    pix, seg = _oracle_image(env, pose, mount, idx)
    idx = slice(None) if idx is None else idx
    assert np.array_equal(gtd["depth_range_pixels"].cpu().numpy()[idx], pix)
    assert np.array_equal(gtd["segmentation_pixels"].cpu().numpy()[idx], seg)
    return pix


def test_gimbal_camera_image_equals_oracle_at_the_link_pose():
    with articulated_cpu_stack():
        torch.manual_seed(0)
        env = _env("base_quadrotor_with_gimbal_camera", "env_with_obstacles", n=4)
        assert env.sensor.robot_state.data_ptr() == env.engine.body_state[:, 2].data_ptr()
        assert env.sensor.robot_state.stride(0) == 3 * 13
        env.reset()
        gtd = env.global_tensor_dict
        gtd["dof_position_setpoint_tensor"][:, 0], gtd["dof_position_setpoint_tensor"][:, 1] = 0.3, 0.6
        for _ in range(5):
            env.step(torch.zeros(4, 4))
        env.render()
        pix = gimbal_camera_check(env)
        assert (pix < 1.0).any()  # something is in view


def test_no_parent_link_reads_the_robot_state_and_the_mount():
    with articulated_cpu_stack():
        torch.manual_seed(0)
        env = _env("base_quadrotor_with_camera", "env_with_obstacles", n=4)
        env.reset()
        env.step(torch.zeros(4, 4))
        env.render()
        gtd = env.global_tensor_dict
        assert env.sensor.robot_state is env.engine.root_state and env.sensor.mount is env.sensor_mount
        pix, seg = _oracle_image(env, gtd["robot_state_tensor"][:, :7].numpy(), env.sensor_mount.numpy())
        assert np.array_equal(gtd["depth_range_pixels"].numpy(), pix) and np.array_equal(gtd["segmentation_pixels"].numpy(), seg)


def _register_link_camera(name, link, base=None):
    from aerial_gym_simulator_b200.config import robot_config as rc
    from aerial_gym_simulator_b200.config.sensor_config import BaseDepthCameraConfig
    from aerial_gym_simulator_b200.registry._core import robot_registry
    from aerial_gym_simulator_b200.robots import ArticulatedMultirotor, BaseMultirotor
    base = base or rc.BaseQuadWithCameraCfg

    class Cam(BaseDepthCameraConfig):
        parent_link = link
        randomize_placement = False
        height, width = 24, 32

    class Cfg(base):
        class sensor_config(base.sensor_config):
            enable_camera = True
            camera_config = Cam
    robot_registry.register(name, ArticulatedMultirotor if hasattr(base, "joint_config") else BaseMultirotor, Cfg)


def test_rigid_robot_camera_on_a_fixed_link_equals_a_base_camera_with_the_link_folded_in():
    _register_link_camera("_test_quad_motor_camera", "motor_0")
    with articulated_cpu_stack():
        torch.manual_seed(0)
        env = _env("_test_quad_motor_camera", "env_with_obstacles", n=4)
        env.reset()
        env.step(torch.zeros(4, 4))
        env.render()
        R, p = env.robot.urdf_model.link_transforms()["motor_0"]
        assert np.array_equal(R, np.eye(3)) and np.allclose(p, [0.13, -0.13, 0.0])
        mount = env.sensor_mount.numpy().copy()
        mount[..., 0:3] += np.asarray(p, np.float32)
        gtd = env.global_tensor_dict
        pix, seg = _oracle_image(env, gtd["robot_state_tensor"][:, :7].numpy(), mount)
        assert np.array_equal(gtd["depth_range_pixels"].numpy(), pix) and np.array_equal(gtd["segmentation_pixels"].numpy(), seg)


def test_unknown_parent_link_raises():
    _register_link_camera("_test_quad_no_such_link", "no_such_link")
    with articulated_cpu_stack():
        with pytest.raises(ValueError, match=r"no_such_link.*base_link"):
            _env("_test_quad_no_such_link", "env_with_obstacles", n=2)


# ---- gimbal levelling ---------------------------------------------------------------------------------------------------------
def gimbal_levelling(env, steps, dev, level=True):
    """hover under lee_attitude_control commanded to roll 0.3 / pitch -0.2 rad; each env step the gimbal's targets are -(roll, pitch)
    of robot_euler_angles (or 0).  -> the camera link's x axis in the world [N,3] and the base's rotation matrices"""
    gtd = env.global_tensor_dict
    n = env.num_envs
    env.spec.enable_disturbance = False
    env.reset()
    st = gtd["robot_state_tensor"]
    st[:, 3:13] = 0.0
    st[:, 6] = 1.0
    gtd["dof_state_tensor"].zero_()
    gtd["dof_position_setpoint_tensor"].zero_()
    act = torch.zeros(n, 4, device=dev)
    act[:, 1], act[:, 2] = 0.3, -0.2  # (thrust, roll, pitch, yaw rate) of lee_attitude_control; thrust 0 = hover
    b = gtd["robot_body_names"].index("pitch_stage_link")
    for _ in range(steps):
        if level:
            e = gtd["robot_euler_angles"]
            wrap = lambda a: torch.remainder(a + np.pi, 2 * np.pi) - np.pi
            gtd["dof_position_setpoint_tensor"][:, 0] = -wrap(e[:, 0])
            gtd["dof_position_setpoint_tensor"][:, 1] = -wrap(e[:, 1])
        env.step(act)
    q = gtd["robot_body_state_tensor"][:, b, 3:7].double().cpu()
    x = torch.stack([1 - 2 * (q[:, 1] ** 2 + q[:, 2] ** 2), 2 * (q[:, 0] * q[:, 1] + q[:, 2] * q[:, 3]),
                     2 * (q[:, 0] * q[:, 2] - q[:, 1] * q[:, 3])], -1)
    return x, gtd["robot_euler_angles"].double().cpu()


# Tolerance of the levelled camera.  The drive is a spring-damper on each stage (balanced: no static load), so with a constant target
# it settles; what is left after 1 s is the lag behind a target that still moves with the base: a target moving at rate r is
# followed with lag 2 zeta / omega r (0.024 s r for roll, 0.023 s r for pitch), plus the staleness of the Euler angles the targets
# come from, one env step (0.01 s in empty_env, 0.1 s in env_with_obstacles).  With the attitude loop settled to |r| < 0.02 rad/s
# the tilt of the optical axis stays below 0.124 s x 0.02 rad/s = 2.5e-3 rad; 5e-3 rad leaves margin (measured: 3.4e-4 rad).
LEVEL_TOL = 5e-3


def levelling_check(env, dev):
    steps = int(round(1.0 / (env.sim_config.sim.dt * env.cfg.env.num_physics_steps_per_env_step_mean)))  # 1 s
    x, e = gimbal_levelling(env, steps, dev)
    roll, pitch = torch.remainder(e[:, 0] + np.pi, 2 * np.pi) - np.pi, torch.remainder(e[:, 1] + np.pi, 2 * np.pi) - np.pi
    assert (roll - 0.3).abs().max() < 0.05 and (pitch + 0.2).abs().max() < 0.05  # the base did tilt
    assert x[:, 2].abs().max().item() < LEVEL_TOL, x[:, 2].abs().max().item()
    x0, e0 = gimbal_levelling(env, steps, dev, level=False)
    pitch0 = torch.remainder(e0[:, 1] + np.pi, 2 * np.pi) - np.pi
    # targets 0: the camera holds q = 0 and tilts with the base; its x axis dips by the base's pitch
    assert (torch.asin(-x0[:, 2]) - pitch0).abs().max().item() < 0.02


def test_gimbal_levels_the_camera():
    with articulated_cpu_stack():
        torch.manual_seed(0)
        levelling_check(_env("base_quadrotor_with_gimbal_camera", "empty_env", n=4), "cpu")
