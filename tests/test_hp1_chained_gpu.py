"""Chained position-task steps that overlap on the device against the same steps run one at a time, bit for bit.

Consecutive single-launch steps are ordered per 32-env tile, not per grid (DESIGN section 5): per-tile claim and done counters, four
monotonic flag / arrival slots and programmatic dependent launch let up to two steps be in flight at once.  Here K steps are enqueued
behind one torch.cuda._sleep, so they run back to back at device speed instead of at the host's enqueue rate; the same inputs are
then run serialised (a synchronize after every step) and through the two-launch path (mid-step event).  Every output must be the
same bits on all three -- an observation refreshed or left stale on the wrong step, a flag read from the wrong slot or a tile started
before its previous step was published would show here -- with one exception, explained at assert_two_launch: after a reset the
two-launch path's roll and yaw (and vehicle_orientation / vehicle_linvel, built on yaw) are rounded differently, and are held to a
bound derived from that cause.  The overlapped and serialised chained runs must also leave the same chain
counters (tile_sync, any_reset[4:16]).

GPU-only, no CPU twin: the tile counters are GPU mechanics (tests/test_gpu_dryrun_cpu.py)."""
import pytest
import torch

from aerial_gym_simulator_b200.hp1 import Hp1Engine
from tests import _hp1_common as H

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
K = 48
SLEEP_CYCLES = 200_000_000  # ~0.1 s at the H100's 1.98 GHz: far longer than the host takes to enqueue K steps
STATE = ("root_state", "motor_thrust", "sim_steps", "episode_count")  # compared after the last step
PER_STEP = ("obs", "reward", "terminations", "truncations", "reset_mask")  # compared after every step
DERIVED = ("euler", "vehicle_orientation", "vehicle_linvel", "body_linvel", "body_angvel")
SCHEDULES = ["quiet", "trunc_last_tile", "crash_only", "all_trunc", "mix"]
ALL_TRUNC_STEP = 10


def inputs(N, schedule):
    """initial state, per-env targets, sim_steps of the schedule, K action tensors on the device"""
    spec = H.spec_for("quad_attitude")
    root, _, params = H.random_inputs(spec, N, seed=N + SCHEDULES.index(schedule))
    g = torch.Generator().manual_seed(1000 + N)
    target = torch.rand(N, 3, generator=g) * 4 - 2
    root[:, 0:3] = target + (torch.randn(N, 3, generator=g) * 0.5).clamp(-1.5, 1.5)
    steps0 = torch.randint(0, 500 - K - 1, (N,), generator=g, dtype=torch.int32)  # nobody is due in the window
    first_last = (N - 1) // 32 * 32  # first env of the last tile
    n_last = N - first_last
    if schedule == "trunc_last_tile":  # the last tile's envs, staggered over the window
        steps0[first_last:] = 500 - (3 + 7 * torch.arange(n_last, dtype=torch.int32)) % (K - 4)
    if schedule == "all_trunc":
        steps0[:] = 500 - ALL_TRUNC_STEP
    if schedule == "mix":  # every fourth env, staggered over steps 5..19, and the crash below
        sel = torch.arange(N) % 4 == 1
        steps0[sel] = 500 - (5 + (torch.arange(N, dtype=torch.int32)[sel] // 4) % 15)
    if schedule in ("crash_only", "mix"):  # the last env starts 7.9 m from its target, flying away at 3 m/s: it crosses 8 m in a few steps
        u = torch.randn(3, generator=g)
        u = u / u.norm()
        root[N - 1, 0:3] = target[N - 1] + 7.9 * u
        root[N - 1, 7:10] = 3.0 * u
    acts = [(torch.rand(N, 4, generator=g) * 2 - 1).to(DEV) for _ in range(K)]
    return spec, root, params, target, steps0, acts


def engine(spec, N, root, params, target, steps0, materialize=True):
    e = Hp1Engine(spec, N, DEV, per_env_params="all", seed=7, materialize_derived=materialize)
    H.load_engine_state(e, root, params)
    e.target_position.copy_(target)
    e.sim_steps.copy_(steps0)
    return e


def run(e, acts, derived=True, mid=None, overlapped=False, probe_at=None, after_enqueue=None):
    """K steps -> the per-step outputs, stacked [K, ...].  Before each step the engine's per-step output pointers (observation,
    reward, flags, reset mask, derived arrays) are aimed at that step's slot: a change of the launch arguments on the host, nothing
    is launched.  overlapped: all steps enqueued behind one sleep, which must still be running when step `probe_at` (default: the
    last) has been enqueued -- the evidence that the steps were queued and then ran back to back.  Otherwise a synchronize follows
    every step.  after_enqueue(i): called after step i has been enqueued."""
    K_ = len(acts)
    keys = PER_STEP + (DERIVED if derived else ())
    ring = {k: torch.zeros((K_,) + tuple(getattr(e, k).shape), dtype=getattr(e, k).dtype, device=DEV) for k in keys}
    pending = True
    if overlapped:
        torch.cuda.synchronize()
        torch.cuda._sleep(SLEEP_CYCLES)
        ev = torch.cuda.Event()
        ev.record()
        probe_at = K_ - 1 if probe_at is None else probe_at
    for i, a in enumerate(acts):
        for k in keys:
            setattr(e._buf, k, ring[k][i].data_ptr())
        e.position_task_step(a, mid_event=mid)
        if overlapped and i == probe_at:
            pending = not ev.query()
        if after_enqueue is not None:
            after_enqueue(i)
        if not overlapped:
            torch.cuda.synchronize()
    e.check()
    e._sync_buffers()
    assert pending, "the sleep ended before the steps were enqueued: they did not run back to back"
    out = {k: getattr(e, k).clone() for k in STATE}
    out.update(ring)
    return out


def chain_counters(e):
    return {"tile_sync": e.tile_sync.clone(), "any_reset[4:16]": e.any_reset[4:16].clone()}


def assert_bits(a, b, what):
    for k in b:
        if not torch.equal(a[k], b[k]):
            diff = (a[k] != b[k]).flatten(1).any(1) if k in PER_STEP + DERIVED else None
            where = f" at steps {diff.nonzero().flatten().tolist()[:8]}" if diff is not None else ""
            raise AssertionError(f"{what}: {k} differs{where}")


# The two-launch path is bit-identical to the chained path except for roll and yaw after a reset, and what is built on yaw.  Cause
# (SASS of hp1_refresh_kernel against hp1_step_kernel<4,true,true,241>, sm_90a, the _build.py flags; nvdisasm -gi attributes each
# instruction to its source line and inline site): the two inline copies of euler_xyz_0_2pi (agx_math.cuh) round
#   cosr_cosp = w*w - x*x - y*y + z*z   and   cosy_cosp = w*w + x*x - y*y - z*z
# differently.  The refresh kernel contracts each into FMUL + 3 FFMA; the chained kernel's epilogue copy (hp1.cu, `d =
# update_states(s)` after a reset) computes the four squares once with FMUL, shares them between the two lines and sums them with
# FADD.  sinr_cosp, siny_cosp and sinp get the same instruction sequence in both, so pitch is identical, and so are the body-frame
# velocities (quat_rotate_inverse of the state's own quaternion).  The two roundings of cos*_cosp differ by at most ~11 float32
# roundings of values <= 1 (11 * 2^-24); atan2 turns an input change dc into an angle change of at most |dc| / r, r = |cos pitch|
# for a unit quaternion; wrapping to [0, 2 pi) and the ssa chain add a few ulps of 2 pi.  The bar below is twice that bound, per env
# (unbounded, so only finiteness is left, at exact gimbal lock).
EPS = 2.0 ** -24
ULP_2PI = 2.0 ** -21  # float32 spacing in [4, 8)


def assert_two_launch(ref, got, what):
    assert_bits(ref, {k: v for k, v in got.items() if k not in ("euler", "vehicle_orientation", "vehicle_linvel")}, what)
    if "euler" not in got:
        return
    e_ref, e_got = ref["euler"].double(), got["euler"].double()
    for k in ("euler", "vehicle_orientation", "vehicle_linvel"):
        assert bool(torch.isfinite(got[k]).all()), f"{what}: {k} not finite"
    assert torch.equal(ref["euler"][..., 1], got["euler"][..., 1]), f"{what}: pitch differs"
    cosp = torch.cos(e_ref[..., 1]).abs()
    tol_angle = 2.0 * (11 * EPS / cosp + 4 * ULP_2PI)  # [K, N]
    d = torch.remainder(e_got - e_ref + torch.pi, 2 * torch.pi) - torch.pi
    r_angle = (d[..., [0, 2]].abs() / tol_angle.unsqueeze(-1)).max()
    # q_veh = (0, 0, sin(yaw / 2), cos(yaw / 2)): half the yaw change, plus sincosf's rounding; -q_veh is the same rotation (yaw at 0 / 2 pi)
    qr, qg = ref["vehicle_orientation"].double(), got["vehicle_orientation"].double()
    dq = torch.minimum((qg - qr).abs().amax(-1), (qg + qr).abs().amax(-1))
    r_q = (dq / (tol_angle / 2 + 4 * EPS)).max()
    # the world velocity turned by yaw: |v| times the yaw change, plus a few roundings of |v|
    vr, vg = ref["vehicle_linvel"].double(), got["vehicle_linvel"].double()
    vn = vr.norm(dim=-1)
    r_v = ((vg - vr).abs().amax(-1) / (vn * (tol_angle + 16 * EPS) + 1e-30)).max()
    n_diff = int((got["euler"] != ref["euler"]).sum())
    print(f"\n{what}: {n_diff} roll / yaw values differ, max |d angle| {float(d.abs().max()):.3e}; err / bound: angle "
          f"{float(r_angle):.3f}, vehicle_orientation {float(r_q):.3f}, vehicle_linvel {float(r_v):.3f}")
    assert max(float(r_angle), float(r_q), float(r_v)) <= 1.0, (what, float(r_angle), float(r_q), float(r_v))


def check_schedule(schedule, out, N):
    """the serialised run did what the schedule is for"""
    term = [out["terminations"][s].nonzero().flatten().tolist() for s in range(K)]
    trunc = [out["truncations"][s].nonzero().flatten().tolist() for s in range(K)]
    resets = [sorted(set(t) | set(r)) for t, r in zip(term, trunc)]
    n_crash = sum(len(t) for t in term)
    if schedule == "quiet":
        assert not any(resets)
    elif schedule == "trunc_last_tile":
        first_last = (N - 1) // 32 * 32
        assert n_crash == 0 and sum(len(r) for r in trunc) == N - first_last
        assert all(i >= first_last for r in trunc for i in r)
    elif schedule == "crash_only":
        busy = [s for s in range(K) if resets[s]]
        assert len(busy) == 1 and term[busy[0]] == [N - 1] and not any(trunc), busy
    elif schedule == "all_trunc":
        assert n_crash == 0 and trunc[ALL_TRUNC_STEP] == list(range(N))
        assert sum(len(r) for r in trunc) == N
    else:  # mix: quiet steps, steps with truncations only, one crash
        assert n_crash == 1 and any(term[s] == [N - 1] for s in range(K))
        assert sum(1 for s in range(K) if not resets[s]) >= 10
        assert sum(1 for s in range(K) if trunc[s] and not term[s]) >= 3


@pytest.mark.parametrize("schedule", SCHEDULES)
@pytest.mark.parametrize("N", [32, 777, 4097, 65536])
def test_overlapped_steps_equal_serialised_steps(N, schedule):
    """32 envs: one CTA, so both steps in flight share the SMs with nothing else; 777: a partial last tile; 65,536: the flagship's
    chained launch at full capacity (on a 132-SM H100)"""
    spec, root, params, target, steps0, acts = inputs(N, schedule)
    ser = engine(spec, N, root, params, target, steps0)
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    assert ser._chain_counts, f"{N} envs do not take the chained path on this {sms}-SM device"
    ref = run(ser, acts)
    check_schedule(schedule, ref, N)

    ov = engine(spec, N, root, params, target, steps0)
    assert_bits(ref, run(ov, acts, overlapped=True), "overlapped vs serialised")
    assert_bits(chain_counters(ser), chain_counters(ov), "overlapped vs serialised chain counters")
    # the flagship's own configuration: no derived arrays, only the observation's body velocities are refreshed
    lean = engine(spec, N, root, params, target, steps0, materialize=False)
    assert_bits(ref, run(lean, acts, derived=False, overlapped=True), "overlapped (no derived arrays) vs serialised")

    # the two-launch path (refresh pass; obs-patch pass without derived arrays): same results as the chained path
    for materialize in (True, False):
        mid = torch.cuda.Event(enable_timing=True)
        mid.record()
        two = engine(spec, N, root, params, target, steps0, materialize=materialize)
        assert_two_launch(ref, run(two, acts, derived=materialize, mid=mid),
                    f"two-launch ({'refresh' if materialize else 'obs-patch'} pass) vs chained")


def test_rebase_between_overlapped_windows():
    """CHAIN_REBASE_STEPS = 20: the counters are rebased before steps 20 and 40.  A rebase drains the stream and zeroes the counters
    (Hp1Engine._rebase_chain), so it can only fall between overlapped windows.  Each window -- steps 0-19, 20-39, 40-47 -- is queued
    behind a sleep of its own (the rebase is followed by one), which must still be running when the window's last step has been
    enqueued.  Results and counters equal a serialised run with the same rebase points."""
    N = 4097
    spec, root, params, target, steps0, acts = inputs(N, "mix")
    ser = engine(spec, N, root, params, target, steps0)
    ov = engine(spec, N, root, params, target, steps0)
    for e in (ser, ov):
        e.CHAIN_REBASE_STEPS = 20
    ref = run(ser, acts)
    check_schedule("mix", ref, N)
    windows, rebase = [], ov._rebase_chain

    def rebase_then_sleep():
        rebase()
        torch.cuda._sleep(SLEEP_CYCLES)
        ev = torch.cuda.Event()
        ev.record()
        windows.append([ev, None])

    def probe(i):
        if i in (39, 47):
            windows[-1][1] = not windows[-1][0].query()

    ov._rebase_chain = rebase_then_sleep
    got = run(ov, acts, overlapped=True, probe_at=19, after_enqueue=probe)
    assert len(windows) == 2 and all(w[1] for w in windows), "a window's sleep ended before its steps were enqueued"
    assert ser._chain_T == ov._chain_T == K % 20
    assert_bits(ref, got, "overlapped vs serialised with rebases")
    assert_bits(chain_counters(ser), chain_counters(ov), "chain counters with rebases")
    assert int(ov.tile_sync.max()) == K % 20
