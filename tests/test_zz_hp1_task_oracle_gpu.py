"""The fused position-task step, hp1_step_kernel<M, TASK=true, COOP, SPEC>, against hp1_oracle run in float64: every one of its nine
instantiations (the seven of hp1.cu's AGX_HP1_SPEC_LIST and the generic <4> / <8>), on the chained single launch (COOP = true) and on
the two-launch path (COOP = false).

Method (as tests/test_hp1_gpu.py::test_fused_position_task_step, with a float64 reference): before every step the oracle state is
rounded to float32 and loaded into the engine (teacher forcing), so each step starts from the same bits on both sides; resets draw
their uniforms from the device RNG's Philox streams (oracle/philox.py).  Bars: 1e-5 of the quantity's scale for root state,
observation, reward, thrust, the reset parameters and the derived arrays; bit-exact terminations, truncations, reset mask, sim_steps
and episode counters.  Envs that fail _hp1_common.well_conditioned are checked for finite values only (and must stay rare).
The Euler angles are compared as angles (the difference wrapped to (-pi, pi]): at roll or yaw = +-pi a float32 chain and a float64
chain may legitimately land on opposite ends of the range.

Paths (hp1.cu: agx_hp1_position_task_step_profiled):
  strict-cooperative          the chained single launch;
  strict-cooperative-derived  the same with the derived arrays materialised;
  strict-refresh_pass         two launches, step kernel then hp1_refresh_kernel (forced by asking for the mid-step event);
  strict-obs_patch_pass       two launches, step kernel then hp1_obs_patch_kernel (forced the same way);
  fresh                       non-strict: one launch of the two-launch kernel, observation always refreshed.
Inputs: per-env nonzero targets; sim_steps staggered so that steps TRUNC_STEPS see truncations and the others none; at CRASH_STEP
the last env (in the last, partial tile) is 8.5 m from its target and crashes while no env truncates -- on the chained path that
flag is raised late, from the epilogue, while the other warps already wait on the arrival count.

Measured worst err / tol (H100 80GB HBM3, 700 W power limit; the module prints it per run under pytest -s): 0.84 with 3 sub-steps
(thrust), 0.70 at 65,537 envs, 0.05-0.52 elsewhere.  The module and tests/test_hp1_chained_gpu.py take about 1 minute together there.

With --gpu-dryrun the same text runs on the host shadow (tests/_cpu_stack.py: CpuHp1Engine), at smaller env counts; the device-only
assertions (which path the launch took, the chained step's error word) are skipped there."""
import os
import re

import numpy as np
import pytest
import torch

from aerial_gym_simulator_b200 import _lib
from aerial_gym_simulator_b200.hp1 import Hp1Engine
from oracle import hp1_oracle as O
from oracle import philox
from tests import _hp1_common as H

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
HP1_CU = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "aerial_gym_simulator_b200", "csrc", "hp1.cu")
F64 = torch.float64
SEED, OFF = 99, 1000
STEPS = 10
TRUNC_STEPS = (1, 4, 7)  # env i truncates at TRUNC_STEPS[j] if i % 8 == 3 * j (and is never due otherwise)
CRASH_STEP = 5
CTAS_PER_SM = 8          # __launch_bounds__(64, 8) of the step kernel
COOP_RESERVE = 32        # CTA slots the chained launch leaves free (hp1.cu: kCoopReserve)
H100_SMS = 132           # the SM count the CPU twin assumes when it decides which path a size would take
PATHS = {  # id -> (strict_stale_obs, materialize_derived, two_launch)
    "strict-cooperative": (True, False, False),
    "strict-cooperative-derived": (True, True, False),
    "strict-refresh_pass": (True, True, True),
    "strict-obs_patch_pass": (True, False, True),
    "fresh": (False, True, False),
}
CPU_N = {777: 97, 4097: 161, 65536: 256, 65537: 257}  # CPU twin: same tile shapes (full / partial last tile), fewer envs
WORST = {}
TAKEN = {}  # (instantiation, path) -> the runs that launched it


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    if WORST:
        print("\nworst err / tol per run (quantity):")
        for k, (r, what) in sorted(WORST.items()):
            print(f"  {k:60s} {r:.3f} ({what})")


def spec_list():
    """[(num_motors, hp_spec_id)] of hp1.cu's AGX_HP1_SPEC_LIST, parsed from its text like tests/_shadow.py lifts it"""
    txt = open(HP1_CU).read()
    body = re.search(r"#define AGX_HP1_SPEC_LIST\(X\)(.*?)\n#else", txt, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body)
    flag = {"AGX_F_USE_RPS": _lib.F_USE_RPS, "AGX_F_MOTOR_RK4": _lib.F_MOTOR_RK4, "AGX_F_DISCRETE_MIX": _lib.F_DISCRETE_MIX,
            "AGX_F_GYROSCOPIC": _lib.F_GYROSCOPIC}
    flag["AGX_SPEC_FLAGS_ALL"] = sum(flag.values())
    out = []
    for m, ctrl, flags in re.findall(r"X\((\d+),\s*AGX_CTRL_(\w+),\s*\(?([A-Z_0-9 |]+?)\)?\)", body):
        f = 0
        for name in flags.split("|"):
            f |= flag[name.strip()]
        out.append((int(m), hp_spec_id(getattr(_lib, "CTRL_" + ctrl), f)))
    return out


def hp_spec_id(controller, flags):
    return (controller & 0xF) | ((flags & 0xF) << 4)


def instantiation(cfg, specs):
    """the (M, SPEC) of the step kernel pick_kernel launches for cfg: a specialised one, or the generic SPEC = -1"""
    key = (cfg.num_motors, hp_spec_id(cfg.controller, cfg.flags))
    return key if key in specs else (cfg.num_motors, -1)


def _n(N):
    return N if DEV != "cpu" else CPU_N.get(N, N)


def _sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count if DEV != "cpu" else H100_SMS


def chained_fits(N):
    """does the chained launch of N envs fit beside the reserved CTA slots?  (hp1.cu: hp1_task_step_is_chained)"""
    grid = max(1, (-(-N // 32) + 1) // 2)
    return _sms() * CTAS_PER_SM - COOP_RESERVE >= grid


def path_taken(eng, path, N):
    """'chained' (COOP kernel) or 'two-launch' (the COOP = false task kernel, with or without a second pass).  On the device this
    is what the engine reports; the intended path must agree with it."""
    strict, _, two_launch = PATHS[path]
    intended = strict and not two_launch and chained_fits(N)
    if DEV != "cpu":
        assert (bool(eng._chain_counts) and not two_launch) == intended, (path, N, _sms(), eng._chain_counts)
    return "chained" if intended else "two-launch"


def make_engine(spec, N, path, physics_steps=1):
    strict, materialize, _ = PATHS[path]
    return Hp1Engine(spec, N, DEV, per_env_params="all", seed=SEED, env_id_offset=OFF, device_rng_reset=True,
                     strict_stale_obs=strict, materialize_derived=materialize, physics_steps=physics_steps)


def _actions(spec, N, g):
    if spec.controller == _lib.CTRL_NONE:
        a = torch.rand(N, spec.num_actions, generator=g) * (spec.max_thrust - spec.min_thrust) * 1.2 + spec.min_thrust - 0.1
        # motor commands are the reference thrusts themselves: keep them out of (0, 5e-3 max_thrust), where sqrt(ref / k) has
        # unbounded slope (_hp1_common.well_conditioned) -- uniform commands would put ~2 % of the envs there every step
        return torch.where(a.abs() < 0.02, a + 0.04, a)
    a = torch.rand(N, spec.num_actions, generator=g) * 2.4 - 1.2
    if spec.controller == _lib.CTRL_FULLY_ACTUATED:
        a[:, 3:7] = torch.randn(N, 4, generator=g)
    return a


ST_FLOATS = ("root", "thrust", "tau_inc", "tau_dec", "k_thrust", "K_pos", "K_vel", "K_rot", "K_angvel", "bounds_min", "bounds_max")


def oracle_state(model, root, params, N):
    st = O.make_state(model, N, F64)
    st.root, st.thrust = root.to(F64), params["thrust"].to(F64)
    for k in ("tau_inc", "tau_dec", "k_thrust", "K_pos", "K_vel", "K_rot", "K_angvel"):
        setattr(st, k, params[k].to(F64))
    return st


def round_to_f32(st):
    """teacher forcing: the step starts from float32 values on both sides"""
    for k in ST_FLOATS:
        setattr(st, k, getattr(st, k).float().to(F64))


def oracle_step(model, st, actions, target, physics_steps, dist, episodes, strict):
    """PositionSetpointTask.step in float64 (hp1_oracle.position_task_step, with the disturbance and sub-step count of the fused step
    and the device RNG's reset draws) -> obs, reward, terminations, truncations, reset mask, well-conditioned envs.  An env is well
    conditioned if every one of its sub-steps is (_hp1_common.well_conditioned) and its final state is not at gimbal lock."""
    N, M = actions.shape[0], model.num_motors
    ok = H.well_conditioned(model, st, actions).numpy()
    if physics_steps == 0:  # no sub-step: the kernel's derived states are those of the state it was given
        st.derived = O.update_states(st.root)
    for i in range(physics_steps):
        if i:
            ok &= H.well_conditioned(model, st, actions).numpy()
        O.physics_step(model, st, actions, dist)
    st.sim_steps = st.sim_steps + 1
    rew, term = O.position_task_reward(st, target, torch.zeros(N, dtype=torch.bool))
    trunc = st.sim_steps > 500
    rmask = term | trunc
    if bool(rmask.any()):
        idx = np.nonzero(rmask.numpy())[0]
        u = philox.reset_uniforms(SEED, OFF + idx, episodes[idx], M)

        def full(k):
            t = torch.zeros((N,) + u[k].shape[1:], dtype=F64)
            t[torch.from_numpy(idx)] = torch.from_numpy(u[k]).to(F64)
            return t

        draws = O.ResetDraws(*(full(k) for k in ("bounds_lo", "bounds_hi", "state", "K_pos", "K_vel", "K_rot", "K_angvel", "tau_inc",
                                                 "tau_dec", "thrust", "k_thrust")))
        O.reset_envs(model, st, rmask, draws)
    if not strict:  # non-strict: derived states always refreshed before the observation
        st.derived = O.update_states(st.root)
    # the Euler angles of the state after the step are an output too (refreshed derived arrays): the same gimbal-lock criterion
    q = st.root[:, 3:7]
    ok &= ((2.0 * (q[:, 3] * q[:, 1] - q[:, 2] * q[:, 0])).abs() < 0.99995).numpy()
    return O.position_task_obs(st, target), rew, term, trunc, rmask, ok


def _np(t):
    return np.asarray(t.detach().cpu() if torch.is_tensor(t) else t, dtype=np.float64)


def close(label, what, got, ref, scale=None, mask=None, angle=False, rtol=H.RTOL):
    """H.assert_close's bar (rtol of max(|ref|, scale)), recording the worst err / tol of the run"""
    got, ref = _np(got), _np(ref)
    keep = np.ones(ref.shape[0], dtype=bool) if mask is None else np.asarray(mask, dtype=bool)
    if not keep.any():
        return
    keep = keep.reshape((-1,) + (1,) * (ref.ndim - 1))
    if scale is None:
        scale = max(float(np.abs(np.where(keep, ref, 0.0)).max()), 1e-30)
    err = np.abs(got - ref)
    if angle:
        err = np.abs(np.remainder(got - ref + np.pi, 2 * np.pi) - np.pi)
    err = np.where(keep, err, 0.0)  # (indices below are env indices)
    tol = rtol * np.maximum(np.abs(ref), scale)
    ratio = err / tol
    worst = float(np.nanmax(np.where(np.isnan(ratio), np.inf, ratio)))
    if worst > WORST.get(label, (-1.0, ""))[0]:
        WORST[label] = (worst, what)
    assert worst <= 1.0, f"{label} {what}: max err / tol {worst:.3f}, max err {np.nanmax(err):.3e} (scale {scale:.3e}) at " \
                         f"{np.argwhere(~(err <= tol))[:3].tolist()}"


QUANT = (("pos", slice(0, 3), None), ("quat", slice(3, 7), 1.0), ("linvel", slice(7, 10), None), ("angvel", slice(10, 13), None))
DERIVED = (("euler", np.pi), ("vehicle_orientation", 1.0), ("vehicle_linvel", None), ("body_linvel", None), ("body_angvel", None))


def run_task(case, path, N, physics_steps=1, disturbance=False, seed=3):
    """STEPS teacher-forced fused steps of N envs on `path`, each checked against oracle_step in float64 -> (instantiation, path)"""
    strict, materialize, two_launch = PATHS[path]
    label = f"{case} {path} N={N}" + (f" ps={physics_steps}" if physics_steps != 1 else "") + (" dist" if disturbance else "")
    N = _n(N)
    spec = H.spec_for(case)
    model = H.oracle_model_from_spec(spec)
    root, _, params = H.random_inputs(spec, N, seed=seed)
    g = torch.Generator().manual_seed(seed + 17)
    target = torch.rand(N, 3, generator=g) * 4 - 2
    root[:, 0:3] = target + (torch.randn(N, 3, generator=g) * 0.8).clamp(-2.5, 2.5)
    st = oracle_state(model, root, params, N)
    r = torch.arange(N) % 8
    st.sim_steps = torch.randint(0, 500 - STEPS - 1, (N,), generator=g, dtype=torch.int32)
    for j, k in enumerate(TRUNC_STEPS):
        st.sim_steps[r == 3 * j] = 500 - k
    ce = N - 1  # the crashing env: last lane of the last tile
    dist = dist_dev = None
    if disturbance:
        model.enable_disturbance, model.prob_apply_disturbance = True, 0.5
        dist = O.draw_disturbance(model, N, generator=g).contiguous()
        dist_dev = dist.to(DEV)
        dist = dist.to(F64)

    eng = make_engine(spec, N, path, physics_steps)
    eng.target_position.copy_(target)
    tgt = target.to(F64)
    specs = spec_list()
    taken = (instantiation(eng.cfg, specs), path_taken(eng, path, N))
    mid = None
    if two_launch and DEV != "cpu":
        mid = torch.cuda.Event(enable_timing=True)
        mid.record()
    episodes = np.zeros(N, dtype=np.int64)
    n_ill = n_trunc_steps = 0
    for step in range(STEPS):
        actions = _actions(spec, N, g)
        if step == CRASH_STEP:
            u = torch.randn(3, generator=g).to(F64)
            u = u / u.norm()
            st.root[ce, 0:3] = tgt[ce] + 8.5 * u  # 0.5 m beyond the crash distance; moving outwards at 0.1 m/s
            st.root[ce, 7:10] = 0.1 * u
        round_to_f32(st)
        H.sync_engine_from_oracle(eng, st)
        eng.position_task_step(actions.to(DEV), disturbance=dist_dev, mid_event=mid)
        obs, rew, term, trunc, rmask, ok = oracle_step(model, st, actions.to(F64), tgt, physics_steps, dist, episodes, strict)
        episodes += rmask.numpy().astype(np.int64)
        # the schedule happened as intended (on the reference: it does not depend on the kernel)
        if step == CRASH_STEP:
            assert int(term.sum()) == 1 and bool(term[ce]) and not trunc.any(), f"step {step}: crash-only step"
        else:
            assert not term.any(), f"step {step}: unexpected crash"
        if step not in TRUNC_STEPS:
            assert not trunc.any(), f"step {step}: unexpected truncation"
        n_trunc_steps += bool(trunc.any())
        torch.cuda.synchronize()
        tag = f"step {step}"
        assert torch.equal(eng.terminations.cpu(), term), f"{tag} terminations"
        assert torch.equal(eng.truncations.cpu(), trunc), f"{tag} truncations"
        assert torch.equal(eng.reset_mask.cpu(), rmask), f"{tag} reset mask"
        assert torch.equal(eng.sim_steps.cpu(), st.sim_steps), f"{tag} sim_steps"
        assert np.array_equal(eng.episode_count.cpu().numpy(), episodes), f"{tag} episode counters"
        close(label, f"{tag} reward", eng.reward, rew, scale=1.0)
        assert torch.isfinite(eng.root_state).all() and torch.isfinite(eng.motor_thrust).all() and torch.isfinite(eng.obs).all()
        n_ill += int((~ok).sum())
        for nm, sl, sc in QUANT:
            close(label, f"{tag} root {nm}", eng.root_state[:, sl], st.root[:, sl], scale=sc, mask=ok)
        close(label, f"{tag} obs target-pos", eng.obs[:, 0:3], obs[:, 0:3], mask=ok)
        for nm, sl, sc in QUANT[1:]:
            close(label, f"{tag} obs {nm}", eng.obs[:, sl], obs[:, sl], scale=sc, mask=ok)
        close(label, f"{tag} thrust", eng.motor_thrust, st.thrust, mask=ok)
        close(label, f"{tag} tau_inc", eng.tau_inc, st.tau_inc, scale=0.01)
        close(label, f"{tag} tau_dec", eng.tau_dec, st.tau_dec, scale=0.01)
        if spec.use_rps:
            close(label, f"{tag} k_thrust", eng.k_thrust, st.k_thrust, scale=1e-5)
        for k in ("K_pos", "K_vel", "K_rot", "K_angvel", "bounds_min", "bounds_max"):
            close(label, f"{tag} {k}", getattr(eng, k), getattr(st, k))
        if materialize:  # derived arrays follow the same stale / refreshed rule as the observation
            for nm, sc in DERIVED:
                close(label, f"{tag} derived {nm}", getattr(eng, nm), st.derived[nm], scale=sc, mask=ok, angle=nm == "euler")
    # ill-conditioned samples are rare.  quadroot_attitude_euler: the band (0, 5e-3 max_thrust) of reference thrusts is 0.05 N wide
    # with its 10 N motors, against 0.01 N for the default quad, at the same hover thrust: ~2.5 % of its env-steps fall in it
    # (each sub-step is a sample)
    assert n_ill <= (0.04 if case == "quadroot_attitude_euler" else 0.01) * STEPS * N * max(1, physics_steps), n_ill
    assert n_trunc_steps == (len(TRUNC_STEPS) if N >= 8 else 1)
    assert int(episodes.sum()) >= 1 + (N + 7) // 8
    if DEV != "cpu":
        eng.check()
        # after the run, the device's own record of the path: the chained launches advanced every tile's claim / done counters and
        # the engine's step index once per step; the two-launch kernels never touch them
        chained = taken[1] == "chained"
        assert eng._chain_T == (STEPS if chained else 0), (eng._chain_T, taken)
        assert bool((eng.tile_sync == (STEPS if chained else 0)).all()), taken
    TAKEN.setdefault(taken, []).append(label)
    return taken


# ---- every case (all nine instantiations) x every path, 777 envs: 24 full tiles and a partial one of 9 ----------------------------
@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("case", H.ALL_CASES)
def test_every_case_and_path(case, path):
    run_task(case, path, 777)


# ---- env counts of the flagship configuration ------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("N", [1, 33, 4097, 65536, 65537])
def test_env_counts(N, path):
    """65,536 envs fill the chained path's capacity on a 132-SM H100 exactly (1,056 - 32 CTA slots); 65,537 need one CTA more and
    take the two-launch path.  The device's SM count decides, and the test says which path ran."""
    inst, taken = run_task("quad_attitude", path, N)
    if DEV != "cpu" and N >= 65536:
        print(f"\n{N} envs, {path}: {_sms()} SMs -> {taken} path")
    if PATHS[path][0] and not PATHS[path][2] and DEV != "cpu" and _sms() == H100_SMS:
        assert taken == ("chained" if N <= 65536 else "two-launch")


# ---- sub-step counts and an explicit disturbance tensor ----------------------------------------------------------------------------
@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("option", ["physics_steps=0", "physics_steps=3", "disturbance"])
@pytest.mark.parametrize("case", ["quad_attitude", "octa_velocity"])
def test_step_options(case, option, path):
    """physics_steps = 0 (no sub-step: the state is kept and the derived states are its own), 3 fused sub-steps, and a disturbance
    wrench given as an [N,6] tensor (half the envs disturbed), added in every sub-step"""
    ps = {"physics_steps=0": 0, "physics_steps=3": 3}.get(option, 1)
    run_task(case, path, 777, physics_steps=ps, disturbance=option == "disturbance", seed=5)


# ---- coverage ------------------------------------------------------------------------------------------------------------------------
def test_every_instantiation_on_both_paths():
    """the oracle runs of this module launched all nine instantiations of the task kernel, each on the chained path and on the
    two-launch path.  What counts is what the runs above recorded (run_task: the instantiation pick_kernel chooses for the engine's
    config, the path confirmed after the run by the device's chain counters); a pair that no run has covered yet -- when this test is
    selected on its own -- is run here, from the (case, path) grid of test_every_case_and_path."""
    specs = spec_list()
    assert len(specs) == 7 and len(set(specs)) == 7, specs
    want = {(i, k) for i in set(specs) | {(4, -1), (8, -1)} for k in ("chained", "two-launch")}
    for case in H.ALL_CASES:
        for path in PATHS:
            if want - set(TAKEN):
                eng = make_engine(H.spec_for(case), _n(777), path)
                if (instantiation(eng.cfg, specs), path_taken(eng, path, _n(777))) not in TAKEN:
                    run_task(case, path, 777)
    missing = sorted(want - set(TAKEN))
    assert not missing, f"not exercised: {missing}"
    print("\n" + "\n".join(f"  <{m}, {s:4d}> {k:10s}: {len(v)} runs, e.g. {v[0]}" for ((m, s), k), v in sorted(TAKEN.items())))
