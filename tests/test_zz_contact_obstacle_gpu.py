"""Contact between free obstacles (args['contact_obstacle_obstacle'], agx_obstacle_obstacle_contact) on the GPU: the kernel against
its host shadow bit for bit in dynamic_env at 1 to 8,192 envs, graph and launch step modes bit-identical over 20 env steps with
resets and env_actions, and the depth image after a collision against the brute-force ray-cast oracle at the corrected poses."""
import random

import numpy as np
import pytest
import torch

from aerial_gym_simulator_b200.hp2 import ContactMotion, obstacle_obstacle_contact
from oracle import hp2_oracle as RO
from tests import _hp2_common as H2
from tests._cpu_stack_obstacle_contact import obstacle_obstacle_shadow
from tests.test_zz_contact_gpu import _env
from tests.test_zz_contact_moving_gpu import _twists, random_twists

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PAIRS = dict(contact_moving_obstacles=True, contact_dynamic_obstacles=True, contact_obstacle_obstacle=True)


@pytest.fixture(autouse=True)
def _needs_the_kernels():
    if DEV == "cpu":  # the CPU dry run of the GPU test text: the robot's contact kernel has no CPU twin
        pytest.skip("the contact kernels have no CPU twin")


def _squeeze(st, seed):
    """the in-play assets of each env pulled towards the env's centroid by up to 60 %, so that many pairs overlap"""
    g = torch.Generator().manual_seed(seed)
    st = st.clone()
    active = st[..., 2] > -500.0
    c = (st[..., 0:3] * active[..., None]).sum(1) / active.sum(1).clamp(min=1)[..., None]
    f = torch.rand(st.shape[:2], generator=g)[..., None] * 0.6
    st[..., 0:3] = torch.where(active[..., None], st[..., 0:3] + (c[:, None] - st[..., 0:3]) * f, st[..., 0:3])
    return st


@pytest.mark.parametrize("n", [1, 127, 129, 4097, 8192])
def test_kernel_equals_shadow_in_dynamic_env(n):
    env = _env("dynamic_env", n=n, seed=60 + n % 7, **PAIRS)
    E, A = env.num_envs, env.num_obs_in_env
    st = random_twists(_squeeze(env.global_tensor_dict["env_asset_state_tensor"].cpu(), 61), seed=62)
    rows = st.to(DEV).contiguous()
    obstacle_obstacle_contact(env.contact_params, ContactMotion(rows, torch.zeros(E, 1, dtype=torch.int32, device=DEV)),
                              env._obstacle_mass, env._obstacle_boxes)
    torch.cuda.synchronize()
    ref = st.numpy().copy()
    count, _ = obstacle_obstacle_shadow(env.contact_params, ref, env._obstacle_mass.table.cpu().numpy(),
                                        env._obstacle_boxes.boxes.cpu().numpy(), env._obstacle_boxes.asset_file.cpu().numpy())
    got = rows.cpu().numpy()
    bad = (got != ref).reshape(E, -1).any(1)
    assert not bad.any(), f"{int(bad.sum())} of {E} envs differ, first {int(np.nonzero(bad)[0][0])}"
    assert (count > 0).mean() > 0.5 and (got != st.numpy()).any()
    if n >= 4097:
        assert (count == 128).any()  # a full list (parked stacks) is exercised too


def test_graph_and_launch_modes_bit_identical_with_obstacle_contact():
    a = _env("dynamic_env", n=77, seed=63, step_mode="graph", contact_obstacle_ground=True, **PAIRS)
    b = _env("dynamic_env", n=77, seed=63, step_mode="launch", contact_obstacle_ground=True, **PAIRS)
    assert a.step_mode == "graph" and b.step_mode == "launch"
    g = torch.Generator(device=DEV).manual_seed(64)
    moved = False
    for step in range(20):
        act = (torch.rand(a.num_envs, a.num_robot_actions, generator=g, device=DEV) * 2 - 1) * 3.0
        tw = _twists(a, g)
        kw = {} if step % 5 == 4 else {"env_actions": tw}
        before = a.global_tensor_dict["env_asset_state_tensor"].clone()
        for env in (a, b):
            random.seed(900 + step)
            env.step(actions=act, **kw)
        torch.cuda.synchronize()
        assert torch.equal(a.engine.root_state, b.engine.root_state), f"step {step}"
        assert torch.equal(a.collision_tensor, b.collision_tensor)
        for k in ("robot_contact_force_tensor", "env_asset_state_tensor"):
            assert torch.equal(a.global_tensor_dict[k], b.global_tensor_dict[k]), f"step {step}: {k}"
        assert torch.equal(a._obj_pose, b._obj_pose) and torch.equal(a.scene.nodes, b.scene.nodes)
        moved |= not torch.equal(before, a.global_tensor_dict["env_asset_state_tensor"])
        if step % 4 == 3:  # resets: fresh (overlapping) obstacle poses in some envs
            ids = torch.arange(step % 7, a.num_envs, 9, device=DEV)
            for env in (a, b):
                torch.manual_seed(1000 + step)
                env.reset_idx(ids)
            assert torch.equal(a.global_tensor_dict["env_asset_state_tensor"], b.global_tensor_dict["env_asset_state_tensor"])
    assert moved and {m for _, m in a._graphs} == {False, True}


def test_depth_image_after_a_collision_equals_the_oracle_at_the_corrected_poses():
    env = _env("dynamic_env", n=33, seed=65, **PAIRS)
    ast = env.global_tensor_dict["env_asset_state_tensor"]
    ast.copy_(_squeeze(ast.cpu(), 66).to(DEV))  # overlapping obstacles: the first sub-step pushes them apart
    env._repose_scene()
    before = ast.clone()
    env.step(actions=torch.zeros(env.num_envs, env.num_robot_actions, device=DEV),
             env_actions=torch.zeros(env.num_envs, env.num_obs_in_env, 6, device=DEV))
    torch.cuda.synchronize()
    assert (ast[..., 7:13].abs().amax(-1) > 0).sum() > 20  # knocked apart (the zero twist leaves only the solve's)
    assert not torch.equal(ast[..., 0:7], before[..., 0:7])
    idx = env._obj_asset.unsqueeze(-1).expand(-1, -1, 7)
    assert torch.equal(env._obj_pose, torch.gather(ast[..., 0:7], 1, idx))  # the scene shows the corrected poses
    env.sensor.capture()
    torch.cuda.synchronize()
    sc, gtd = env.scene, env.global_tensor_dict
    tris, segs, cnt = RO.build_world_tris(env._obj_pose.cpu().numpy(), sc.obj_template.cpu().numpy(), sc.obj_seg_counter.cpu().numpy(),
                                          sc.tmpl_tri_offset.cpu().numpy(), sc.tmpl_tris.cpu().numpy(), sc.tmpl_seg_base.cpu().numpy(),
                                          sc.tmpl_seg_mask.cpu().numpy(), sc.K * sc.L)
    so, _ = H2.oracle_sensor(env.sensor_cfg)
    ref_pix, _ = RO.cast(so, gtd["robot_state_tensor"][:, :7].cpu().numpy(), env.sensor_mount.cpu().numpy(), None, tris, segs, cnt)
    assert np.array_equal(gtd["depth_range_pixels"].cpu().numpy(), ref_pix)
