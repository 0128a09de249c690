"""The reference arm of bench.py (oracle/reference_arm.py: the reference's own, unmodified control stack from baseline/_ref + the
oracle integrator) against the oracle port on the same state and actions: the arm that is TIMED as "the reference" computes what
the parity oracle computes.  Skips where the reference was never staged (baseline/_ref is built by __graft_entry__.build() in the
build container and travels with the snapshot).  The checks run in a fresh interpreter: importing the reference's `aerial_gym`
must not meet the product's `compat` alias of the same name that other tests install."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_REF = os.environ.get("AERIAL_GYM_REFERENCE", "")
_HAVE = os.path.isdir(os.path.join(ROOT, "baseline", "_ref", "aerial_gym", "registry")) or bool(_REF and os.path.isdir(os.path.join(_REF, "aerial_gym")))
pytestmark = pytest.mark.skipif(not _HAVE, reason="reference not staged (baseline/_ref)")


@pytest.mark.parametrize("check", ["check_steps_like_the_oracle_port", "check_resets_with_the_reference_reset"])
def test_reference_arm(check):
    r = subprocess.run([sys.executable, os.path.abspath(__file__), check], capture_output=True, text=True, cwd=ROOT, timeout=300)
    assert r.returncode == 0 and "CHECK_OK" in r.stdout, (r.stdout[-1500:], r.stderr[-1500:])


def check_steps_like_the_oracle_port():
    n = 96
    task = R.ReferencePositionTask(n, seed=3)
    mm = task.robot.control_allocator.motor_model
    model = task.model
    st = O.make_state(model, n)
    g = torch.Generator().manual_seed(11)
    root = task.gtd["robot_state_tensor"]
    q = torch.randn(n, 4, generator=g)
    root[:, 0:3] = torch.randn(n, 3, generator=g)
    root[:, 3:7] = q / q.norm(dim=1, keepdim=True)
    root[:, 7:13] = torch.randn(n, 6, generator=g)
    st.root = root.clone()
    st.thrust = mm.current_motor_thrust.clone()
    st.tau_inc, st.tau_dec = mm.motor_time_constants_increasing.clone(), mm.motor_time_constants_decreasing.clone()
    st.k_thrust = mm.motor_thrust_constant.clone()
    c = task.robot.controller
    st.K_pos, st.K_vel = c.K_pos_tensor_current.clone(), c.K_linvel_tensor_current.clone()
    st.K_rot, st.K_angvel = c.K_rot_tensor_current.clone(), c.K_angvel_tensor_current.clone()
    task.sim_steps[:] = 0
    tgt = torch.zeros(n, 3)
    for step in range(6):
        a = torch.rand(n, 4, generator=g) * 2 - 1
        obs_r, rew_r, crash_r, trunc_r = task.step(a.clone())
        obs_o, rew_o, crash_o, trunc_o, rmask = O.position_task_step(model, st, a, tgt, draw_fn=None)
        assert not rmask.any()
        assert torch.equal(crash_r, crash_o) and torch.equal(trunc_r, trunc_o)
        scale = max(1.0, float(obs_o.abs().max()))
        assert (obs_r - obs_o).abs().max().item() <= 1e-5 * scale, f"step {step}"
        assert (rew_r - rew_o).abs().max().item() <= 1e-5 * max(1.0, float(rew_o.abs().max()))
        assert (root - st.root).abs().max().item() <= 1e-5 * scale


def check_resets_with_the_reference_reset():
    n = 32
    task = R.ReferencePositionTask(n, seed=4, episode_len_steps=3)
    a = torch.zeros(n, 4)
    for _ in range(3):
        task.step(a)
    assert not task.truncations.any()
    before = task.gtd["robot_state_tensor"].clone()
    task.step(a)  # sim_steps = 4 > 3: everybody truncates and is reset by BaseMultirotor.reset_idx
    assert task.truncations.all() and (task.sim_steps == 0).all()
    after = task.gtd["robot_state_tensor"]
    assert (after[:, 0:3].abs() <= 1.0).all() and not torch.equal(before, after)  # inside the +-1 m env bounds of empty_env


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    import torch  # noqa: F401

    from oracle import hp1_oracle as O  # noqa: F401
    from oracle import reference_arm as R  # noqa: F401

    globals().update(torch=torch, O=O, R=R)
    globals()[sys.argv[1]]()
    print("CHECK_OK")
