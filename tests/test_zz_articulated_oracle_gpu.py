"""The articulated step on the H100 against the float64 reference of one whole sub-step (oracle/articulated_oracle.py: substep),
in all four instantiations of articulated_step_kernel<M, NB>: M = 4 / 8 motors, per-body scratch for up to 9 / 16 bodies.

Each case is one physics_step(physics_steps=1) of Hp1Engine(..., articulation=...), compared with AO.substep on the engine's own
float32 inputs: root_state, dof_state, motor_thrust and the five derived outputs.  Tolerance (tests/test_articulated_cpu.py,
section 7): the ABA's bar, 2e-4 of max |(a0, qdd)| of the env, carried through one dt into v, w and qd and through dt^2 into x,
the quaternion and q, plus 8 float32 ulps of the quantity's magnitude for the rounding of the update itself; thrust and derived
outputs at the HP1 bar (1e-5, tests/_hp1_common.py).  Envs that fail _hp1_common.well_conditioned, or whose reference q' lies
within 1e-5 of a joint limit (rounding may take either branch of the projection there), are checked for finite values only.
Measured worst case over this module, err / tol (largest |err|):
                 x     quat  v     w     q            qd           thrust       derived
  host shadow    0.04  0.13  0.00  0.05  0.50 (2e-6) 0.56 (2e-4)  0.36 (7e-6)  <= 0.05
  H100 (kernel)  0.04  0.12  0.00  0.06  0.33 (8e-6) 0.34 (7e-4)  0.34 (7e-6)  <= 0.05
(H100 80GB HBM3; the module printed these at its end under pytest -s.)  Wall time on the H100: 41 s for the 53 tests.

With --gpu-dryrun the same text runs on the host shadow (CpuArticulatedHp1Engine)."""
import numpy as np
import pytest
import torch

from aerial_gym_simulator_b200.hp1 import Hp1Engine
from oracle import hp1_oracle as HO
from tests import _hp1_common as H
from tests._cpu_stack_articulated import CpuArticulatedHp1Engine
from tests.test_articulated_cpu import (check_derived, check_substep, load_inputs, morphy_compliant, near_limit, reference_substep,
                                        shaped_art, substep_inputs, table_of)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ART_THREADS = 128  # kArtThreads of articulated.cu: the block size whose ragged last block the env counts below exercise
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    print("\nworst err / tol (worst |err|) per quantity: " + ", ".join(f"{k} {v[0]:.2f} ({v[1]:.1e})" for k, v in sorted(WORST.items())))


def _engine(*a, **k):
    return Hp1Engine(*a, **k) if DEV != "cpu" else CpuArticulatedHp1Engine(*a, **k)


def _spec(M, **over):
    spec = H.spec_for("quad_attitude" if M == 4 else "octa_velocity")
    for k, v in over.items():
        setattr(spec, k, v)
    return spec


def sample_envs(N, k=512, seed=0):
    """env 0, the last env, both sides of eight block boundaries spread over N, then seeded random envs up to k (all envs if N <= k)"""
    if N <= k:
        return np.arange(N)
    s = {0, N - 1}
    for b in np.unique(np.linspace(ART_THREADS, N - 1, 8).astype(int) // ART_THREADS * ART_THREADS):
        s |= {int(b) - 1, int(b)}
    rest = np.setdiff1d(np.arange(N), list(s))
    return np.sort(np.concatenate([list(s), np.random.default_rng(seed).choice(rest, k - len(s), replace=False)]))


def limit_joints(art, rng, every=2):
    """every `every`-th joint gets limits lower in [-0.8, -0.3], upper in [0.3, 0.8]"""
    b = art.bodies
    for i in range(1, b.num_bodies, every):
        b.limited[i], b.lower[i], b.upper[i] = True, -rng.uniform(0.3, 0.8), rng.uniform(0.3, 0.8)
    return art


def run_case(spec, art, N, seed, per_env_params="all", idx=None, prepare=None):
    """one sub-step of N envs on the engine, the reference on envs idx (default: sample_envs) -> (engine, inputs, reference, ok, idx)"""
    eng = _engine(spec, N, DEV, per_env_params=per_env_params, articulation=art)
    inp = substep_inputs(spec, art, N, seed)
    if prepare is not None:
        prepare(inp)
    load_inputs(eng, inp)
    eng.physics_step(inp["actions"].to(DEV), disturbance=inp["dist"].to(DEV), physics_steps=1)
    torch.cuda.synchronize()
    idx = sample_envs(N, seed=seed) if idx is None else idx
    ref, ok = reference_substep(eng, spec, art, inp, idx)
    return eng, inp, ref, ok, idx


def check_properties(eng):
    """every env: finite state, unit quaternion, every limited joint inside its limits"""
    for t in (eng.root_state, eng.dof_state, eng.motor_thrust):
        assert bool(torch.isfinite(t).all())
    assert float((eng.root_state[:, 3:7].norm(dim=1) - 1).abs().max()) < 1e-6
    tab = table_of(eng.art)
    D = eng.dof_state.shape[1]
    lim = torch.tensor(tab["limited"][1:D + 1].astype(bool), device=eng.dof_state.device)
    lo = torch.tensor(tab["lower"][1:D + 1], dtype=torch.float32, device=eng.dof_state.device)
    hi = torch.tensor(tab["upper"][1:D + 1], dtype=torch.float32, device=eng.dof_state.device)
    q = eng.dof_state[..., 0]
    assert not bool((lim & ((q < lo) | (q > hi))).any())


# ---- every instantiation: tree size x motors x tree shape, motor placement, drives on / off, per-env or constant parameters ----
TREES = [(B, M, shape) for B in (1, 2, 9, 10, 16) for M in (4, 8) for shape in (("chain",) if B <= 2 else ("chain", "star", "random"))]


@pytest.mark.parametrize("B,M,shape", TREES)
def test_every_instantiation_matches_reference(B, M, shape):
    """B = 9 / 10 sit on either side of the NB switch.  Motors: all on the base, on the leaves, or all but one on the last body
    (cycled over the three shapes, so every (B, M) of 9+ bodies sees all three).  Two launches per tree: drive on with one of
    per_env_params "all" / "auto", drive off with the other."""
    i = TREES.index((B, M, shape))
    motors = ("base", "leaves", "cluster")[("chain", "star", "random").index(shape)] if B > 2 else "cluster"
    params = ("all", "auto") if i % 2 else ("auto", "all")
    for drive, pep in zip((True, False), params):
        rng = np.random.default_rng(1000 + 10 * i + drive)
        art = limit_joints(shaped_art(rng, B, shape, M=M, drive=drive, motors=motors), rng, every=3)
        eng, inp, ref, ok, idx = run_case(_spec(M), art, 64, 10 * i + drive, per_env_params=pep)
        assert (eng.tau_dec is None) == (pep == "auto")  # "auto" reads a constant motor parameter from the config
        assert ok.mean() > 0.8
        assert check_substep(eng, _spec(M), inp, ref, ok, idx, WORST) <= 2


# ---- env counts: ragged last blocks, and 65,536 envs ---------------------------------------------------------------------------
@pytest.mark.parametrize("N", [1, 127, 129, 4097])
@pytest.mark.parametrize("M,B", [(4, 9), (8, 16)])
def test_env_counts(N, M, B):
    rng = np.random.default_rng(N + M)
    art = limit_joints(shaped_art(rng, B, "random", M=M), rng)
    eng, inp, ref, ok, idx = run_case(_spec(M), art, N, N + M)
    assert check_substep(eng, _spec(M), inp, ref, ok, idx, WORST) <= max(2, len(idx) // 100)
    check_properties(eng)


@pytest.mark.parametrize("M", [4, 8])
def test_65536_envs(M):
    """<M, 16>: the reference on 512 sampled envs (env 0, the last, both sides of block boundaries), properties on all"""
    N = 65536
    rng = np.random.default_rng(77 + M)
    art = limit_joints(shaped_art(rng, 13, "random", M=M), rng)
    eng, inp, ref, ok, idx = run_case(_spec(M), art, N, 77 + M)
    sides = set(idx.tolist())
    assert len(idx) == 512 and idx[0] == 0 and idx[-1] == N - 1
    assert sum(b % ART_THREADS == 0 and b - 1 in sides for b in sides) >= 8  # both sides of at least eight block boundaries
    assert check_substep(eng, _spec(M), inp, ref, ok, idx, WORST) <= 5
    check_properties(eng)


# ---- controllers ---------------------------------------------------------------------------------------------------------------
QUAD = ["quad_attitude", "quad_position", "quad_velocity", "quad_acceleration", "quad_rates", "quad_none", "quad_velocity_steering"]


@pytest.mark.parametrize("case", QUAD + ["octa_fully_actuated", "octa_velocity"])
def test_controllers(case):
    """the seven quad controllers on morphy_compliant (<4, 9>); fully-actuated and velocity control of an octarotor on a 12-body tree
    (<8, 16>).  Thrust against float64 hp1_oracle; ill-conditioned envs (_hp1_common.well_conditioned) checked for finite values."""
    spec = H.spec_for(case)
    if spec.num_motors == 4:
        _, art = morphy_compliant()
    else:
        rng = np.random.default_rng(5)
        art = limit_joints(shaped_art(rng, 12, "random", M=8), rng)
    eng, inp, ref, ok, idx = run_case(spec, art, 256, 300 + QUAD.index(case) if case in QUAD else 320)
    assert ok.mean() > 0.9
    assert check_substep(eng, spec, inp, ref, ok, idx, WORST) <= 3


# ---- limits and continuous joints ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,B", [(4, 10), (8, 9)])
def test_limits_and_continuous_joints(M, B):
    """odd joints limited, their q' crossing the lower limit, the upper limit, or neither (|qd| of 10-40 rad/s: 0.1-0.4 rad per
    sub-step); even joints continuous at |q| of 40-200 rad (range reduction of sincosf in axis_angle).  A crossing joint is clamped
    to its limit exactly and keeps no velocity pointing out of the range."""
    N = 1024
    rng = np.random.default_rng(90 + M)
    art = shaped_art(rng, B, "random", M=M)
    b = art.bodies
    odd = np.arange(1, B) % 2 == 1
    b.limited[1:] = odd
    b.lower[1:] = np.where(odd, -rng.uniform(0.2, 0.5, B - 1), 0.0)
    b.upper[1:] = np.where(odd, rng.uniform(0.2, 0.5, B - 1), 0.0)

    def prepare(inp):
        r = np.random.default_rng(91 + M)
        dof = inp["dof"].numpy()
        lo, hi = b.lower[1:].astype(np.float32), b.upper[1:].astype(np.float32)
        dof[..., 0] = np.where(odd, lo + (hi - lo) * r.uniform(0, 1, (N, B - 1)), r.choice([-1, 1], (N, B - 1)) * r.uniform(40, 200, (N, B - 1)))
        dof[..., 1] = np.where(odd, r.choice([-1, 1], (N, B - 1)) * r.uniform(10, 40, (N, B - 1)), dof[..., 1])

    eng, inp, ref, ok, idx = run_case(_spec(M), art, N, 92 + M, prepare=prepare)
    skipped = check_substep(eng, _spec(M), inp, ref, ok, idx, WORST)
    assert skipped <= len(idx) // 100, skipped
    tab = table_of(eng.art)
    lo, hi = tab["lower"][1:B], tab["upper"][1:B]
    qf = ref["q_free"][:, odd]
    below, above = qf < lo[odd] - 1e-5, qf > hi[odd] + 1e-5
    inside = (qf > lo[odd] + 1e-5) & (qf < hi[odd] - 1e-5)
    assert below.sum() >= 50 and above.sum() >= 50 and inside.sum() >= 50, (below.sum(), above.sum(), inside.sum())
    got = eng.dof_state.cpu().double().numpy()[idx][:, odd]
    keep = (ok & ~near_limit(tab, ref))[:, None]
    assert (got[..., 0] == lo[odd])[below & keep].all() and (got[..., 1] >= 0)[below & keep].all()
    assert (got[..., 0] == hi[odd])[above & keep].all() and (got[..., 1] <= 0)[above & keep].all()
    cont = np.abs(inp["dof"].numpy()[idx][:, ~odd, 0])
    assert cont.min() >= 40 and cont.max() <= 200
    check_properties(eng)


# ---- damping factors and velocity caps -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,B", [(4, 16), (8, 10)])
def test_damping_and_velocity_caps(M, B):
    """linear / angular damping 0.5, caps 0.6 m/s and 0.9 rad/s just below the start speeds (|v| in 0.5-0.7, |w| in 0.8-1.0)"""
    spec = _spec(M, linear_damping=0.5, angular_damping=0.5, max_linear_velocity=0.6, max_angular_velocity=0.9)
    rng = np.random.default_rng(60 + M)
    art = shaped_art(rng, B, "random", M=M)
    N = 256

    def prepare(inp):
        r = np.random.default_rng(61 + M)
        for sl, lo, hi in ((slice(7, 10), 0.5, 0.7), (slice(10, 13), 0.8, 1.0)):
            d = r.normal(size=(N, 3))
            inp["root"][:, sl] = torch.tensor(d / np.linalg.norm(d, axis=1, keepdims=True) * r.uniform(lo, hi, (N, 1)), dtype=torch.float32)

    eng, inp, ref, ok, idx = run_case(spec, art, N, 62 + M, prepare=prepare)
    vn, wn = np.linalg.norm(ref["root"][:, 7:10], axis=1), np.linalg.norm(ref["root"][:, 10:13], axis=1)
    assert (vn > 0.6 - 1e-9).sum() >= 10 and (vn < 0.59).sum() >= 10 and (wn > 0.9 - 1e-9).sum() >= 10 and (wn < 0.89).sum() >= 10
    assert check_substep(eng, spec, inp, ref, ok, idx, WORST) == 0


# ---- step counts, per instantiation --------------------------------------------------------------------------------------------
INSTANTIATIONS = [(4, 9), (4, 16), (8, 9), (8, 16)]


def _art_for(M, NB, seed):
    rng = np.random.default_rng(seed)
    return limit_joints(shaped_art(rng, NB if NB == 9 else 14, "random", M=M), rng)


@pytest.mark.parametrize("M,NB", INSTANTIATIONS)
def test_zero_physics_steps(M, NB):
    """physics_steps = 0: the state is left bit for bit, the derived outputs are update_states of it"""
    N, spec, art = 200, _spec(M), _art_for(M, NB, 7)
    eng = _engine(spec, N, DEV, per_env_params="all", articulation=art)
    inp = substep_inputs(spec, art, N, 8)
    load_inputs(eng, inp)
    before = [t.clone() for t in (eng.root_state, eng.dof_state, eng.motor_thrust)]
    eng.physics_step(inp["actions"].to(DEV), disturbance=inp["dist"].to(DEV), physics_steps=0)
    torch.cuda.synchronize()
    for a, t in zip(before, (eng.root_state, eng.dof_state, eng.motor_thrust)):
        assert torch.equal(a, t)
    d = {k: v.numpy() for k, v in HO.update_states(inp["root"].double()).items()}
    model, st = H.oracle_model_from_spec(spec), HO.make_state(H.oracle_model_from_spec(spec), N, torch.float64)
    st.root = inp["root"].double()
    check_derived(eng, d, np.arange(N), H.well_conditioned(model, st, inp["actions"].double()).numpy(), WORST)


@pytest.mark.parametrize("M,NB", INSTANTIATIONS)
def test_ten_steps_in_one_launch_equal_ten_launches(M, NB):
    """physics_steps = 10 in one launch is bit-identical to 10 launches of one sub-step"""
    N, spec, art = 300, _spec(M), _art_for(M, NB, 9)
    inp = substep_inputs(spec, art, N, 10)
    a, b = (_engine(spec, N, DEV, per_env_params="all", articulation=art) for _ in range(2))
    for e in (a, b):
        load_inputs(e, inp)
    act, dist = inp["actions"].to(DEV), inp["dist"].to(DEV)
    a.physics_step(act, disturbance=dist, physics_steps=10)
    for _ in range(10):
        b.physics_step(act, disturbance=dist, physics_steps=1)
    torch.cuda.synchronize()
    for k in ("root_state", "dof_state", "motor_thrust", "euler", "vehicle_orientation", "vehicle_linvel", "body_linvel", "body_angvel"):
        assert torch.equal(getattr(a, k), getattr(b, k)), k
    assert bool(torch.isfinite(a.root_state).all())
