"""The task-epilogue kernels on the H100 against float64 references, at their edges and on every launch shape: the ten C entries
(12 kernels, 13 instantiations counting lidar_nav_pool_kernel<VEC4 = true / false>) that produce the rewards, crash flags and
observations of the navigation, LiDAR / radar navigation, motor-command (e2e) and setpoint sim2real tasks, and the IMU.

Reference: the oracles' own torch code (oracle/aux_oracle.py, lidar_nav_oracle.py, e2e_task_oracle.py, sim2real_oracle.py; pinned to
the reference task code by their fixtures) run on float64 copies of the kernel's own float32 inputs.  Parameters are the float32
values the kernel receives.  Each case mixes seeded random envs with envs built to sit on an edge (EDGES below: angles at 0,
2 pi +- 1 ulp and +-pi, pitch within 1e-4 of pi/2, qw = +-0, distances at 0, at a threshold and equal to the previous distance,
clipping thresholds, zero velocity, exp arguments that underflow), and every env is compared.

Tolerance, per output and per env.  e = 8 float32 ulps of 1 (8 x 2^-23).  A term mag * exp(-ex v^2) is off by at most e |mag|
from rounding inside it, plus its largest slope |mag| sqrt(2 ex / E) (|mag| ex for exp(-ex |v|)) times the error of v; a
computed distance or rotated vector is off by e x (the magnitudes of the vectors it was computed from); a difference of two
such distances multiplied by a gain g (closer / towards_goal: 400..1200 in s2r, 10..100 in e2e, 10 in nav) is off by
g e (dist + prev_dist) -- the cancellation's condition number; an angle from atan2(y, x) is off by e / hypot(x, y), one from
asin(s) by min(e / sqrt(1 - s^2), sqrt(2 e)); an ssa / wrapped angle by e (|a| + 2 pi); a rotation-6d or quaternion built from
angles by 2 x the sum of the angles' errors.  Every bound is summed over the terms of the output (written out next to each comparison
below).  Copies (actions, velocities, LiDAR columns, untouched columns, the in-place quaternion, pos_error_prev) are compared bit
for bit.

Branch outputs (crash flags, the IMU clamp, the pool's clipping side, the s2r acceleration variant's dist < prev_dist choice that
shows in the reward, the LiDAR reward's stable / vdc > 0 choices) must equal the reference's decision, except where the float64
value lies within the float32 rounding band (its bound above) of the threshold; there either side is accepted and the env is
counted (EXEMPT).  The threshold constructions (position 0, identity frame, axis-aligned target or return) are exact in float32
too, so they are never exempt: they must take the reference's side.  The pool runs once with invalid_value == max_range (the
tasks' setting) and once with -1, where clipping at max_range shows in the pooled image.  Angles whose ssa lands within the band of +-pi may come out on either side of the wrap (a quaternion built
from them may come out negated).  Envs whose bound exceeds 0.5 (atan2 of two near-zero arguments at exact gimbal lock) are checked
for the reference's finite / non-finite pattern only, and counted.  test_zz_exemptions_are_rare_and_every_edge_ran asserts that
every (entry, edge) pair ran and that exempt envs stay under 1 % per entry and decision; it skips when only part of the
module was selected.

Measured worst err / tol (largest |err|) on an H100 80GB HBM3 (power limit 700 W), printed at the end of the module under pytest -s:
  nav_reward   pos_error 0.18 (4e-5)  reward 0.05 (4e-3)        nav_obs   dir 0.03  dist 0.10  angles 0.06
  imu          meas 0.42 (7e-5)       bias 0.09                 lnav_pool image_ds 0.14 (1e-6)  ttc 0.02
  lnav_reward  pos_error 0.33 (3e-6)  reward 0.02 (2e-5)        lnav_obs  dir 0.04  dist 0.13  angles 0.06  yaw_error 0.05
  e2e_reward   reward 0.03 (1e-4)                               e2e_obs   pos 0.12  rot6d 0.02 (5e-5)
  s2r_reward   reward 0.03 (2e-3)     act_vehicle 0.05          s2r_obs   pos 0.12  quat 0.01 (2e-4)  vel 0.08
Exempt envs, of about 70,000 per entry: at most 50 per decision (s2r closer side), 43 ill-conditioned (s2r reward).  No float32
|R20| of the e2e observation rounded past 1 here (asin_domain 0).  Wall time on the H100: 17 s for the 82 tests.

With --gpu-dryrun the same text runs on the host shadow build (tests/csrc/host_shadow.cu: the same *_core.cuh text)."""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

from aerial_gym_simulator_b200 import _lib
from oracle import aux_oracle as A
from oracle import e2e_task_oracle as E
from oracle import hp1_oracle as O
from oracle import lidar_nav_oracle as L
from oracle import sim2real_oracle as S

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
G = os.path.join(os.path.dirname(__file__), "golden")
ENV_THREADS = 128  # kAuxThreads / kEnvThreads of the per-env kernels: the block whose ragged last block the env counts exercise
NS = [1, 127, 128, 129, 4097, 65537]
EPS = 8 * 2.0 ** -23
F32_2PI = float(np.float32(2 * math.pi))
SENTINEL = -1234.5
WORST, EXEMPT, COVER, DONE = {}, {}, set(), set()

EDGES = {
    "nav_reward": ["dist_0", "dist_eq_prev", "exp_underflow", "qw_0", "crash", "q_neg", "ragged"],
    "nav_obs": ["angle_0", "angle_2pi_pm_ulp", "angle_pm_pi", "dist_0", "qw_0", "q_neg", "obs_pad", "ragged"],
    "imu": ["clamp_at_max", "clamp_beyond", "qw_0", "q_neg", "gravity", "world_frame", "body_frame", "ragged"],
    "lnav_pool": ["at_max_range", "at_min_range", "ulp_past_thresholds", "zero_return", "far_return", "zero_velocity", "invalid_ne_max_range", "vec4",
                  "scalar",
                  "trailing_rows_cols", "pool_h_eq_H", "pool_w_1", "bands_gt_warps", "smem_gt_48k", "vec4_vs_scalar"],
    "lnav_reward": ["dist_0", "dist_1", "dist_3", "vel_0", "vdc_0", "angle_0", "angle_2pi_pm_ulp", "angle_pm_pi", "ttc_underflow",
                    "crash", "radar", "q_neg", "pos_error_prev", "ragged"],
    "lnav_obs": ["angle_0", "angle_2pi_pm_ulp", "angle_pm_pi", "dist_0", "lidar_null", "obs_pad", "q_neg", "ragged"],
    "e2e_reward": ["dist_0", "dist_at_crash", "dist_eq_prev", "exp_underflow", "qw_0", "target_null", "crash_in", "q_neg", "ragged"],
    "e2e_obs": ["pitch_lock", "qw_0", "angle_pm_pi", "target_null", "obs_pad", "q_neg", "ragged"],
    "s2r_reward": ["dist_10_pm_ulp", "dist_eq_prev", "dist_0", "angle_0", "angle_2pi_pm_ulp", "angle_pm_pi", "pitch_lock", "qw_0",
                   "target_null", "act_out_null", "crash_in", "q_neg", "ragged"],
    "s2r_obs": ["qw_0", "qw_neg0", "q_neg", "angle_0", "angle_2pi_pm_ulp", "angle_pm_pi", "pitch_lock", "target_null", "obs_pad",
                "ragged"],
}


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    print("\nworst err / tol (worst |err|) per entry and output:")
    for k, v in sorted(WORST.items()):
        print(f"  {k[0]:12s} {k[1]:18s} {v[0]:.3f} ({v[1]:.1e})")
    print("exempt envs per entry and decision: " + ", ".join(f"{k[0]}.{k[1]} {v[0]}/{v[1]}" for k, v in sorted(EXEMPT.items())))


@pytest.fixture(autouse=True)
def _done(request):
    yield
    DONE.add(request.node.name)


# ---- plumbing --------------------------------------------------------------------------------------------------------------------
def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _dev(t):
    return t.to(DEV, copy=True).contiguous()  # always a copy: in / out buffers must not alias the inputs kept for the reference


def f32(x):
    return torch.as_tensor(np.asarray(x, dtype=np.float32))


def _ulps(x, k):
    """x moved by k float32 ulps (k may be negative)"""
    x = np.asarray(x, np.float32)
    for _ in range(abs(k)):
        x = np.nextafter(x, np.float32(np.inf if k > 0 else -np.inf))
    return x


def _unit_quats(n, g):
    q = torch.randn(n, 4, generator=g, dtype=torch.float64)
    return (q / q.norm(dim=1, keepdim=True)).float()


def _quat_from_euler64(r, p, y):
    return O.quat_from_euler_xyz(torch.as_tensor(r, dtype=torch.float64), torch.as_tensor(p, dtype=torch.float64),
                                 torch.as_tensor(y, dtype=torch.float64)).float()


def _edge_rows(N, names, seed, reps=3):
    """env rows for each edge: disjoint, random over all N (so they also land in ragged last blocks); with fewer envs than edges,
    which edges get a row rotates with the seed"""
    rng = np.random.default_rng(seed)
    k = min(N, len(names) * reps)
    rows = rng.permutation(N)[:k]
    order = np.roll(np.arange(len(names)), seed % len(names))
    out = {n: [] for n in names}
    for i, r in enumerate(rows):
        out[names[order[i % len(names)]]].append(int(r))
    return {n: torch.tensor(v, dtype=torch.long) for n, v in out.items() if v}


def _cover(entry, *edges):
    for e in edges:
        assert e in EDGES[entry], (entry, e)
        COVER.add((entry, e))


def _exempt(entry, decision, near, total=None):
    n = int(near.sum()) if torch.is_tensor(near) else int(near)
    t = EXEMPT.setdefault((entry, decision), [0, 0])
    t[0] += n
    t[1] += int(total if total is not None else near.numel())


def compare(entry, name, got, ref, tol, wrap=None, sign_flip=None):
    """got (float32) against ref (float64) within tol (float64, broadcast).  A reference non-finite value must be matched by the same
    class (nan / same-signed inf).  Rows with tol > 0.5 are checked for that pattern only (counted as ill_conditioned).
    wrap: bool rows whose angle may come out 2 pi away; sign_flip: bool rows whose quaternion may come out negated."""
    got, ref = got.double(), ref.double()
    tol = torch.as_tensor(tol, dtype=torch.float64).expand_as(ref).clone()
    fin = torch.isfinite(ref)
    same_nf = (got.isnan() & ref.isnan()) | (got == ref)
    assert bool((fin | same_nf).all()), (entry, name, "non-finite pattern differs", got[~(fin | same_nf)][:5], ref[~(fin | same_nf)][:5])
    ill = tol > 0.5
    if ill.dim() > 1:
        ill_rows = ill.any(dim=tuple(range(1, ill.dim())))
        _exempt(entry, "ill_conditioned", ill_rows)
    else:
        _exempt(entry, "ill_conditioned", ill)
    err = torch.where(fin, (got - ref).abs(), torch.zeros_like(ref))
    if wrap is not None:
        w = wrap.view(-1, *([1] * (ref.dim() - 1))).expand_as(ref)
        err = torch.where(w & fin, torch.minimum(err, ((got - ref).abs() - 2 * math.pi).abs()), err)
    if sign_flip is not None:
        alt = (got + ref).abs().amax(dim=1, keepdim=True).expand_as(ref)
        row = (got - ref).abs().amax(dim=1, keepdim=True).expand_as(ref)
        s = sign_flip.view(-1, 1).expand_as(ref)
        err = torch.where(s & fin & (alt < row), (got + ref).abs(), err)
    assert bool(torch.isfinite(got[fin & ~ill]).all()), (entry, name, "kernel non-finite where the reference is finite")
    ratio = torch.where(ill | ~fin | (err == 0), torch.zeros_like(err), err / tol)
    worst = float(ratio.max()) if ratio.numel() else 0.0
    i = int(ratio.argmax()) if ratio.numel() else 0
    abs_err = float(err[~ill & fin].max()) if bool((~ill & fin).any()) else 0.0
    w = WORST.setdefault((entry, name), (0.0, 0.0))
    WORST[(entry, name)] = (max(w[0], worst), max(w[1], abs_err))
    assert worst <= 1.0, (entry, name, worst, "got", float(got.flatten()[i]), "ref", float(ref.flatten()[i]), "tol", float(tol.flatten()[i]),
                          "at", np.unravel_index(i, ref.shape))


def decision(entry, name, got, ref, near):
    """a branch decision: got == ref except where the float64 value lies within the rounding band of the threshold (counted)"""
    bad = (got != ref) & ~near
    assert not bool(bad.any()), (entry, name, torch.nonzero(bad)[:5].flatten().tolist())
    _exempt(entry, name, near)


def bits(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def same(a, b):
    """equal values, nan where nan (a zero may change sign)"""
    return torch.allclose(a, b, rtol=0, atol=0, equal_nan=True)


def slope(mag, ex):
    """largest |d/dv| of mag * exp(-ex v^2)"""
    return abs(mag) * math.sqrt(2.0 * abs(ex) / math.e)


def ssa_wrap_near(a_ref):
    """rows whose ssa lies within the band of +-pi (either side of the wrap is accepted)"""
    return (math.pi - a_ref.abs()) <= EPS * (a_ref.abs() + 2 * math.pi) * 4


def _state(N, stride, g, pos=None, q=None, vel=None):
    st = torch.randn(N, stride, generator=g).float()
    if pos is not None:
        st[:, 0:3] = pos
    st[:, 3:7] = _unit_quats(N, g) if q is None else q
    if vel is not None:
        st[:, 7:10] = vel
    return st


def _stride(N):
    return 13 if N % 2 == 0 else 17  # robot_state_stride > 13 on the odd env counts


# ---- NavigationTask reward / obs (hp1_aux.cu) --------------------------------------------------------------------------------------
def _nav_params():
    d = np.load(os.path.join(G, "nav_task_epilogue.npz"))
    vals = np.asarray(d["param_values"], np.float32)
    p = _lib.AgxNavRewardParams()
    for i, v in enumerate(vals):
        p.v[i] = float(v)
    return p, {k: float(v) for k, v in zip(A.NAV_PARAM_NAMES, vals)}


def _nav_inputs(N, seed):
    g = torch.Generator().manual_seed(seed)
    pos = torch.randn(N, 3, generator=g) * 4
    target = pos + torch.randn(N, 3, generator=g) * torch.rand(N, 1, generator=g) * 6
    yaw = torch.rand(N, generator=g, dtype=torch.float64) * 2 * math.pi
    veh = _quat_from_euler64(torch.zeros(N), torch.zeros(N), yaw)
    inp = dict(pos=pos, veh=veh, target=target, prev_err=torch.randn(N, 3, generator=g) * 3, crashes=(torch.rand(N, generator=g) < 0.05),
               act=torch.rand(N, 4, generator=g) * 2 - 1, prev_act=torch.rand(N, 4, generator=g) * 2 - 1,
               euler=torch.rand(N, 3, generator=g) * 2 * math.pi, blv=torch.randn(N, 3, generator=g), bav=torch.randn(N, 3, generator=g),
               u_vec=torch.rand(N, 3, generator=g), u_euler=torch.rand(N, 3, generator=g))
    return inp, g


def _angle_edges(inp, rows, key, cols):
    """angle_0 / angle_2pi_pm_ulp / angle_pm_pi on inp[key][:, cols]"""
    pi32 = np.float32(math.pi)
    vals = {"angle_0": [0.0, -0.0], "angle_2pi_pm_ulp": [_ulps(F32_2PI, -1), _ulps(F32_2PI, 1), F32_2PI, _ulps(0.0, -1)],
            "angle_pm_pi": [pi32, -pi32, _ulps(pi32, -1), _ulps(-pi32, 1), np.float32(3 * math.pi)]}
    for name, vs in vals.items():
        if name in rows:
            for j, r in enumerate(rows[name].tolist()):
                for c in cols:
                    inp[key][r, c] = float(vs[(j + c) % len(vs)])


@pytest.mark.parametrize("N", NS)
def test_nav_reward(N):
    entry = "nav_reward"
    inp, g = _nav_inputs(N, 100 + N)
    rows = _edge_rows(N, EDGES[entry][:-1], N)
    if "dist_0" in rows:
        inp["target"][rows["dist_0"]] = inp["pos"][rows["dist_0"]]
    if "dist_eq_prev" in rows:  # identity vehicle frame and position 0: err == target exactly, prev_dist == dist
        r = rows["dist_eq_prev"]
        inp["veh"][r] = f32([0, 0, 0, 1])
        inp["pos"][r] = 0.0
        inp["prev_err"][r] = inp["target"][r]
    if "exp_underflow" in rows:
        r = rows["exp_underflow"]
        inp["target"][r] = inp["pos"][r] + 400.0
        inp["act"][r], inp["prev_act"][r] = 1e3, -1e3
    if "qw_0" in rows:
        inp["veh"][rows["qw_0"]] = f32([0, 0, 1, 0])
    if "crash" in rows:
        inp["crashes"][rows["crash"]] = True
    if "q_neg" in rows:
        inp["veh"][rows["q_neg"]] *= -1
    _cover(entry, *rows.keys(), *(["ragged"] if N % ENV_THREADS else []))
    params, p = _nav_params()
    frac = float(np.float32(0.37))
    stride = _stride(N)
    g2 = torch.Generator().manual_seed(N)
    st = _state(N, stride, g2, pos=inp["pos"])

    def run(veh):
        lib = _lib.load()
        pe, pp, rew = _dev(inp["prev_err"]), torch.full((N, 3), SENTINEL, device=DEV), torch.full((N,), SENTINEL, device=DEV)
        t = [_dev(x) for x in (st, veh, inp["target"], inp["crashes"].to(torch.uint8), inp["act"], inp["prev_act"])]
        _lib.check(lib.agx_nav_reward(N, _p(t[0]), stride, _p(t[1]), _p(t[2]), _p(t[3]), _p(t[4]), _p(t[5]), frac, C.byref(params), _p(pe),
                                      _p(pp), _p(rew), None), "agx_nav_reward")
        torch.cuda.synchronize()
        return rew.cpu(), pe.cpu(), pp.cpu()

    rew, pe, pp = run(inp["veh"])
    d = {k: v.double() for k, v in inp.items() if v.is_floating_point()}
    err = A.nav_pos_error(d["veh"], d["target"], d["pos"])
    ref = A.nav_compute_reward(err, d["prev_err"], inp["crashes"], d["act"], d["prev_act"], frac, p)
    assert bits(pp, inp["prev_err"])  # pos_error_prev: the value pos_error held on entry, bit for bit
    scale = d["target"].norm(dim=1) + d["pos"].norm(dim=1)
    compare(entry, "pos_error", pe, err, EPS * scale.unsqueeze(1))
    dist, prev = err.norm(dim=1), d["prev_err"].norm(dim=1)
    dd = EPS * (scale + dist)
    k, mult = p["getting_closer_reward_multiplier"], 1 + 2 * frac
    exps = [(p[a], p[b]) for a, b in zip(A.NAV_PARAM_NAMES[0:4:2], A.NAV_PARAM_NAMES[1:4:2])]
    pens = [(p[A.NAV_PARAM_NAMES[i]], p[A.NAV_PARAM_NAMES[i + 1]]) for i in range(5, 17, 2)]
    ab = (d["act"].abs() + d["prev_act"].abs())[:, [0, 2, 3, 0, 2, 3]]
    tol = mult * (sum(EPS * abs(m) + slope(m, x) * dd for m, x in exps) + 2 * abs(k) * (dd + EPS * (prev + dist)) + dd / 20 + EPS * (1 + dist / 20))
    tol = tol + sum(EPS * abs(m) + slope(m, x) * EPS * ab[:, i] for i, (m, x) in enumerate(pens)) + EPS * ref.abs()
    compare(entry, "reward", rew, ref, tol)
    crashed = inp["crashes"]
    assert bool((rew[crashed] == float(np.float32(p["collision_penalty"]))).all())
    if N >= 129:  # q against -q: quat_rotate_inverse is quadratic in q, the kernel's outputs are bit-identical
        rew2, pe2, _ = run(-inp["veh"])
        assert same(rew2, rew) and same(pe2, pe)  # (equal values: a zero may change sign)
        _cover(entry, "q_neg")


@pytest.mark.parametrize("N", NS)
def test_nav_obs(N):
    entry = "nav_obs"
    inp, g = _nav_inputs(N, 200 + N)
    rows = _edge_rows(N, EDGES[entry][:-2], N + 1)
    _angle_edges(inp, rows, "euler", (0, 1))
    if "dist_0" in rows:
        inp["target"][rows["dist_0"]] = inp["pos"][rows["dist_0"]]
        inp["u_vec"][rows["dist_0"][::2]] = 0.0
    if "qw_0" in rows:
        inp["veh"][rows["qw_0"]] = f32([0, 0, 1, 0])
    if "q_neg" in rows:
        inp["veh"][rows["q_neg"]] *= -1
    stride, obs_stride = _stride(N), 17 + 3 + N % 5
    _cover(entry, *rows.keys(), *(["obs_pad"] if obs_stride > 17 else []), *(["ragged"] if N % ENV_THREADS else []))
    st = _state(N, stride, torch.Generator().manual_seed(N), pos=inp["pos"])

    def run(veh):
        lib = _lib.load()
        obs = torch.full((N, obs_stride), SENTINEL, device=DEV)
        t = [_dev(x) for x in (st, veh, inp["euler"], inp["blv"], inp["bav"], inp["act"], inp["target"], inp["u_vec"], inp["u_euler"])]
        _lib.check(lib.agx_nav_obs(N, _p(t[0]), stride, *[_p(x) for x in t[1:]], _p(obs), obs_stride, None), "agx_nav_obs")
        torch.cuda.synchronize()
        return obs.cpu()

    obs = run(inp["veh"])
    d = {k: v.double() for k, v in inp.items() if v.is_floating_point()}
    ref = A.nav_process_obs(d["veh"], d["pos"], d["target"], d["euler"], d["blv"], d["bav"], d["act"], d["u_vec"], d["u_euler"])
    vec = O.quat_rotate_inverse(d["veh"], d["target"] - d["pos"])
    dist = vec.norm(dim=1)
    dv = EPS * (d["target"].norm(dim=1) + d["pos"].norm(dim=1) + dist)
    # pert / dist: relative error of pert (e |vec| + 0.2 e) and of dist, over dist
    t_dir = (dv + EPS * 0.2) / dist + ref[:, 0:3].abs().amax(dim=1) * (dv / dist + EPS)
    compare(entry, "dir", obs[:, 0:3], ref[:, 0:3], t_dir.unsqueeze(1))
    compare(entry, "dist", obs[:, 3], ref[:, 3], dv)
    a = d["euler"][:, 0:2]
    compare(entry, "angles", obs[:, 4:6], ref[:, 4:6], EPS * (a.abs() + 2 * math.pi + 0.1), wrap=ssa_wrap_near(O.ssa(a)).any(dim=1))
    _exempt(entry, "ssa_wrap", ssa_wrap_near(O.ssa(a)).any(dim=1))
    assert bits(obs[:, 6], torch.zeros(N)) and bits(obs[:, 7:17], torch.cat([inp["blv"], inp["bav"], inp["act"]], 1))
    assert bool((obs[:, 17:] == SENTINEL).all())  # the VAE-latent columns and the stride padding keep their bits
    if N >= 129:
        assert same(run(-inp["veh"]), obs)
        _cover(entry, "q_neg")


# ---- IMU (hp1_aux.cu) ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", NS)
def test_imu(N):
    entry = "imu"
    g = torch.Generator().manual_seed(300 + N)
    world, comp = N % 2 == 1, N % 4 == 1
    cfg = _lib.AgxImuConfig()
    cfg.world_frame, cfg.enable_noise, cfg.enable_bias = int(world), int(N != 128), int(N != 127)
    sqrt_dt = float(np.float32(0.1))
    cfg.sqrt_dt = sqrt_dt
    grav = f32([0.0, 0.0, -9.81])
    gw = grav * (0.0 if comp else 1.0)
    for i in range(3):
        cfg.g_world[i] = float(gw[i])
    noise_std, bias_std, max_meas = f32([0.02] * 3 + [0.003] * 3), f32([0.01] * 3 + [0.001] * 3), f32([40.0] * 3 + [8.0] * 3)
    for i in range(6):
        cfg.noise_std[i], cfg.bias_std[i], cfg.max_meas[i] = float(noise_std[i]), float(bias_std[i]), float(max_meas[i])
    fs, stride = 6, _stride(N)
    force = torch.randn(N, fs, generator=g) * 30
    mass = torch.rand(N, generator=g) * 1.5 + 0.5
    st = _state(N, stride, g)
    bav = torch.randn(N, 3, generator=g) * 4
    sq = _unit_quats(N, g)
    nn, nb, bias = torch.randn(N, 6, generator=g), torch.randn(N, 6, generator=g), torch.randn(N, 6, generator=g) * 0.05
    rows = _edge_rows(N, ["clamp_at_max", "clamp_beyond", "qw_0", "q_neg"], N + 2)
    for name in ("clamp_at_max", "clamp_beyond"):
        if name in rows:  # identity rotations, unit mass, no noise / bias: the measurement is force - g exactly
            r = rows[name]
            st[r, 3:7], sq[r], mass[r] = f32([0, 0, 0, 1]), f32([0, 0, 0, 1]), 1.0
            nn[r], nb[r], bias[r] = 0.0, 0.0, 0.0
            force[r, 0] = float(max_meas[0]) * (1 if name == "clamp_at_max" else 2) * torch.tensor([1.0, -1.0]).repeat(len(r))[:len(r)]
            bav[r, 0] = float(max_meas[3]) * (1 if name == "clamp_at_max" else 2)
    if "qw_0" in rows:
        st[rows["qw_0"], 3:7] = f32([0.6, 0, 0.8, 0])
        sq[rows["qw_0"][::2]] = f32([0, 0.6, 0.8, 0])
    if "q_neg" in rows:
        st[rows["q_neg"], 3:7] *= -1
    _cover(entry, *rows.keys(), *(["gravity"] if not comp else []), "world_frame" if world else "body_frame")
    if N % ENV_THREADS:
        _cover(entry, "ragged")

    def run(state):
        lib = _lib.load()
        b, meas = _dev(bias), torch.full((N, 6), SENTINEL, device=DEV)
        t = [_dev(x) for x in (force, mass, state, bav, sq, nn, nb)]
        _lib.check(lib.agx_imu_update(N, C.byref(cfg), _p(t[0]), fs, _p(t[1]), _p(t[2]), stride, _p(t[3]), _p(t[4]), _p(t[5]), _p(t[6]), _p(b),
                                      _p(meas), None), "agx_imu_update")
        torch.cuda.synchronize()
        return meas.cpu(), b.cpu()

    meas, b_new = run(st)
    D = lambda t: t.double()
    ref, ref_b = A.imu_update(D(force), D(mass), D(st[:, 3:7]), D(bav), D(sq), D(grav), world, comp, D(bias), D(nn), D(nb), D(noise_std), D(bias_std),
                              D(max_meas), sqrt_dt ** 2, enable_noise=bool(cfg.enable_noise), enable_bias=bool(cfg.enable_bias))
    compare(entry, "bias", b_new, ref_b, EPS * (D(bias).abs() + (D(nb) * D(bias_std)).abs() * sqrt_dt))
    acc_in = (D(force[:, 0:3]) / D(mass).unsqueeze(1)).norm(dim=1, keepdim=True) + 9.81
    unclamped = torch.cat([acc_in.expand(N, 3), D(bav).norm(dim=1, keepdim=True).expand(N, 3)], 1)
    tol = EPS * (2 * unclamped + cfg.enable_bias * 2 * ref_b.abs() + cfg.enable_noise * (D(nn) * D(noise_std)).abs() / sqrt_dt)
    # the clamp's side: the unclamped float64 value against +-max_meas
    v = A.imu_update(D(force), D(mass), D(st[:, 3:7]), D(bav), D(sq), D(grav), world, comp, D(bias), D(nn), D(nb), D(noise_std), D(bias_std),
                     torch.full((6,), 1e30, dtype=torch.float64), sqrt_dt ** 2, enable_noise=bool(cfg.enable_noise), enable_bias=bool(cfg.enable_bias))[0]
    near = ((v.abs() - D(max_meas)).abs() <= tol)
    decision(entry, "clamp", meas.abs() == max_meas, v.abs() >= D(max_meas), near)
    compare(entry, "meas", meas, ref, tol)
    if N >= 129:  # q against -q (the robot's): quat_mul negates q_ws exactly, both rotations are quadratic
        st2 = st.clone()
        st2[:, 3:7] *= -1
        m2, b2 = run(st2)
        assert same(m2, meas) and same(b2, b_new)
        _cover(entry, "q_neg")


# ---- LiDAR navigation: pooling (lidar_nav.cu, both instantiations) ----------------------------------------------------------------
MAXR, MINR = float(np.float32(10.0)), float(np.float32(0.2))
POOL_SHAPES = [  # (envs, H, W, pool_h, pool_w)
    (4, 48, 120, 3, 6),    # the reference's shape: 16 bands over 8 warps, VEC4
    (3, 7, 13, 3, 6),      # trailing rows and columns, scalar
    (3, 8, 12, 3, 5),      # trailing rows and columns, VEC4
    (3, 6, 8, 6, 1),       # pool_h == H, pool_w == 1, VEC4
    (2, 5, 9, 5, 1),       # pool_h == H, pool_w == 1, scalar
    (2, 40, 4, 2, 4),      # 20 bands over 8 warps
    (3, 1, 40, 1, 7),      # one row
    (2, 8, 300, 2, 3),     # 57.6 KB of band staging: past the 48 KB line, VEC4
    (2, 9, 301, 2, 6),     # past the 48 KB line, scalar, trailing row and column
    (1, 1, 2133, 1, 1),    # exactly 200 KB of staging: the largest accepted band
]


def _vec4(H, W, ph, aligned):  # the entry's rule for lidar_nav_pool_kernel<true>
    return aligned and (ph * W * 3) % 4 == 0 and (H * W * 3) % 4 == 0


def _pool_inputs(n, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    pos = torch.round(torch.randn(n, 3, generator=g) * 16) / 8  # dyadic: an axis-aligned offset from it is exact
    pos[:, 2] = 0.0
    vel = torch.randn(n, 3, generator=g) * 3
    vel[0] = 0.0  # env 0 stands still: every return takes ttc_max
    dirs = torch.randn(n, H, W, 3, generator=g, dtype=torch.float64)
    dirs = dirs / dirs.norm(dim=-1, keepdim=True)
    rng = torch.rand(n, H, W, 1, generator=g, dtype=torch.float64) * 12 + 0.02
    pc = (pos.double().view(n, 1, 1, 3) + dirs * rng).float()
    flat = pc.view(n, -1, 3)
    m = torch.rand(flat.shape[:2], generator=g)
    z = lambda v: torch.stack([torch.zeros_like(v), torch.zeros_like(v), v], -1)  # along +z from pos (pos.z = 0): exact
    e = pos.view(n, 1, 3).expand_as(flat)
    pick = lambda lo, hi: (m >= lo) & (m < hi)
    for lo, hi, r in ((0.00, 0.02, MAXR), (0.02, 0.04, MINR), (0.04, 0.05, float(_ulps(MAXR, 1))), (0.05, 0.06, float(_ulps(MAXR, -1))),
                      (0.06, 0.07, float(_ulps(MINR, 1))), (0.07, 0.08, float(_ulps(MINR, -1))), (0.08, 0.10, 0.0)):
        s = pick(lo, hi)
        flat[s] = (e + z(torch.full(flat.shape[:2], r)))[s]
    far = pick(0.10, 0.13)
    flat[far] = (e + torch.randn(flat.shape, generator=g) * 300)[far]  # invalid: far beyond max_range
    return pc, pos, vel


def _pool_run(pc, pos, vel, ph, pw, offset, invalid):
    lib = _lib.load()
    n, H, W, _ = pc.shape
    raw = torch.zeros(pc.numel() + 8, device=DEV)
    pcd = raw[offset:offset + pc.numel()].view(n, H, W, 3)
    pcd.copy_(pc.to(DEV))
    st = torch.zeros(n, 14, device=DEV)
    st[:, 0:3], st[:, 7:10], st[:, 6] = pos.to(DEV), vel.to(DEV), 1.0
    ds = torch.full((n, H // ph, W // pw), SENTINEL, device=DEV)
    ttc = torch.full((n,), SENTINEL, device=DEV)
    _lib.check(lib.agx_lidar_nav_pool(n, H, W, ph, pw, _p(pcd), _p(st), 14, MAXR, MINR, invalid, MAXR, _p(ds), _p(ttc), None), "agx_lidar_nav_pool")
    torch.cuda.synchronize()
    return ds.cpu(), ttc.cpu()


@pytest.mark.parametrize("inv", [MAXR, -1.0])  # -1: a return clipped at max_range no longer looks like one at max_range
@pytest.mark.parametrize("n,H,W,ph,pw", POOL_SHAPES)
def test_lidar_nav_pool(n, H, W, ph, pw, inv):
    entry = "lnav_pool"
    pc, pos, vel = _pool_inputs(n, H, W, H * 1000 + W)
    ds, ttc = _pool_run(pc, pos, vel, ph, pw, 0, inv)
    ds1, ttc1 = _pool_run(pc, pos, vel, ph, pw, 1, inv)  # the same data 4 bytes off: lidar_nav_pool_kernel<false>
    assert bits(ds, ds1) and bits(ttc, ttc1)  # both instantiations: bit-identical
    _cover(entry, "vec4_vs_scalar")
    d = pc.double() - pos.double().view(n, 1, 1, 3)
    r = d.norm(dim=-1)
    want_ds, want_ttc = L.pool(pc.double(), pos.double(), vel.double(), (ph, pw), max_range=MAXR, min_range=MINR, invalid_value=inv, ttc_max=MAXR)
    # clipping side: a return within the rounding band of max_range / min_range may be clipped either way
    band = EPS * r
    near_px = ((r - MAXR).abs() <= band) | ((r - MINR).abs() <= band)
    near_px &= (d[..., 0] != 0) | (d[..., 1] != 0)  # returns straight above pos (the threshold constructions) are computed exactly
    OH, OW = H // ph, W // pw
    near_w = near_px[:, :OH * ph, :OW * pw].reshape(n, OH, ph, OW, pw).any(4).any(2)
    decision(entry, "clip_side", ds == inv, want_ds == inv, near_w)
    tol_ds = torch.where(near_w, torch.full_like(want_ds, 1e9), EPS * want_ds.abs())
    compare(entry, "image_ds", ds, want_ds, tol_ds)
    # time to collision: per return t = rc / (vc + 1e-6) for vc > 0; vc off by e |vel|, rc by e rc
    rc = torch.where((r > MAXR) | (r < MINR), inv, r)
    vc = (vel.double().view(n, 1, 1, 3) * d / (r.unsqueeze(-1) + 1e-6)).sum(-1)
    t = torch.where(vc > 0, rc / (vc + 1e-6), torch.full_like(rc, MAXR))
    dt = torch.where(vc > 0, t.abs() * (EPS * vel.double().norm(dim=1).view(n, 1, 1) / (vc + 1e-6) + 2 * EPS), torch.zeros_like(t)) + near_px * 1e9
    cand = (t - dt) <= want_ttc.view(n, 1, 1)
    tol_t = torch.where(cand, dt, torch.zeros_like(dt)).flatten(1).amax(1)
    tol_t = torch.where(((t + dt) < 0).flatten(1).any(1), torch.zeros_like(tol_t), tol_t)  # surely negative: the clamp gives 0 exactly
    compare(entry, "ttc", ttc, want_ttc, torch.minimum(tol_t, torch.full_like(tol_t, 1e9)) + EPS * MAXR)
    assert float(ttc[0]) == MAXR
    ulp_r = torch.tensor([float(_ulps(MAXR, 1)), float(_ulps(MAXR, -1)), float(_ulps(MINR, 1)), float(_ulps(MINR, -1))], dtype=torch.float64)
    present = {"at_max_range": r == MAXR, "at_min_range": r == MINR, "ulp_past_thresholds": torch.isin(r, ulp_r), "zero_return": r == 0,
               "far_return": r > 2 * MAXR, "zero_velocity": vel.abs().sum(1) == 0, "invalid_ne_max_range": torch.tensor(inv != MAXR)}
    _cover(entry, *[k for k, v in present.items() if bool(v.any())])
    if H % ph or W % pw:
        _cover(entry, "trailing_rows_cols")
    if ph == H:
        _cover(entry, "pool_h_eq_H")
    if pw == 1:
        _cover(entry, "pool_w_1")
    if -(-H // ph) > 8:
        _cover(entry, "bands_gt_warps")
    if 8 * ((ph * W * 3 + 3) & ~3) * 4 > 48 * 1024:
        _cover(entry, "smem_gt_48k")
    _cover(entry, "vec4" if _vec4(H, W, ph, True) else "scalar")


# ---- LiDAR navigation: reward and obs (lidar_nav.cu) ------------------------------------------------------------------------------
def _lnav_params(radar):
    d = np.load(os.path.join(G, "lidar_nav_task_epilogue.npz"))
    vals = np.asarray(d["param_values"], np.float32)
    p = _lib.AgxLidarNavRewardParams()
    for i, v in enumerate(vals):
        p.v[i] = float(v)
    p.radar_variant = int(radar)
    return p, {k: float(v) for k, v in zip(L.LIDAR_NAV_PARAM_NAMES, vals)}


def _lnav_inputs(N, seed):
    inp, g = _nav_inputs(N, seed)
    inp["veh"] = _unit_quats(N, g)
    inp["target_yaw"] = (torch.rand(N, generator=g) * 2 - 1) * math.pi
    inp["vlv"] = torch.randn(N, 3, generator=g) * 2
    inp["ttc"] = torch.rand(N, generator=g) * 3
    inp["target"][: N // 3] = inp["pos"][: N // 3] + torch.randn(N // 3, 3, generator=g) * 0.4  # a third within ~1 m (stable)
    return inp, g


@pytest.mark.parametrize("N", NS)
def test_lidar_nav_reward(N):
    entry, radar = "lnav_reward", N % 2 == 0
    inp, g = _lnav_inputs(N, 400 + N)
    names = ["dist_0", "dist_1", "dist_3", "vel_0", "vdc_0", "angle_0", "angle_2pi_pm_ulp", "angle_pm_pi", "ttc_underflow", "crash", "q_neg"]
    rows = _edge_rows(N, names, N + 3)
    _angle_edges(inp, rows, "euler", (2,))
    for name in ("angle_0", "angle_2pi_pm_ulp", "angle_pm_pi"):
        if name in rows:
            inp["target_yaw"][rows[name][::2]] = float(np.float32(math.pi))
    if "dist_0" in rows:
        inp["target"][rows["dist_0"]] = inp["pos"][rows["dist_0"]]
    for name, x in (("dist_1", 1.0), ("dist_3", 3.0), ("vdc_0", 1.0)):
        if name in rows:  # identity frame, position 0: err == target exactly
            r = rows[name]
            inp["veh"][r], inp["pos"][r] = f32([0, 0, 0, 1]), 0.0
            inp["target"][r] = f32([[x, 0, 0], [float(_ulps(x, -1)), 0, 0], [0, 0, float(_ulps(x, 1))]]).repeat(len(r), 1)[:len(r)]
            if name == "vdc_0":
                inp["target"][r] = f32([x, 0, 0])
                inp["vlv"][r] = f32([0, 0.7, -0.3])  # perpendicular: vdc == 0 exactly
    if "vel_0" in rows:  # standing still, and 1e-6 m/s straight at a goal 5 m ahead (where vden's 1e-6 halves vdc)
        r = rows["vel_0"]
        inp["vlv"][r] = 0.0
        r = r[1::2]
        inp["veh"][r], inp["pos"][r], inp["target"][r], inp["vlv"][r] = f32([0, 0, 0, 1]), 0.0, f32([5, 0, 0]), f32([1e-6, 0, 0])
    if "ttc_underflow" in rows:
        inp["ttc"][rows["ttc_underflow"]] = 10.0
    if "crash" in rows:
        inp["crashes"][rows["crash"]] = True
    if "q_neg" in rows:
        inp["veh"][rows["q_neg"]] *= -1
    _cover(entry, *rows.keys(), "pos_error_prev")
    if radar:
        _cover(entry, "radar")
    if N % ENV_THREADS:
        _cover(entry, "ragged")
    params, p = _lnav_params(radar)
    frac = float(np.float32(0.6))
    stride = _stride(N)
    st = _state(N, stride, torch.Generator().manual_seed(N), pos=inp["pos"])

    def run(veh):
        lib = _lib.load()
        pe, pp, rew = _dev(inp["prev_err"]), torch.full((N, 3), SENTINEL, device=DEV), torch.full((N,), SENTINEL, device=DEV)
        t = [_dev(x) for x in (st, veh, inp["target"], inp["euler"], inp["target_yaw"], inp["vlv"], inp["bav"], inp["crashes"].to(torch.uint8),
                               inp["act"], inp["prev_act"], inp["ttc"])]
        _lib.check(lib.agx_lidar_nav_reward(N, _p(t[0]), stride, *[_p(x) for x in t[1:]], frac, C.byref(params), _p(pe), _p(pp), _p(rew), None),
                   "agx_lidar_nav_reward")
        torch.cuda.synchronize()
        return rew.cpu(), pe.cpu(), pp.cpu()

    rew, pe, pp = run(inp["veh"])
    d = {k: v.double() for k, v in inp.items() if v.is_floating_point()}
    ref, err = L.rewards_and_errors(d["veh"], d["pos"], d["target"], d["euler"], d["target_yaw"], d["vlv"], d["bav"], inp["crashes"], d["act"],
                                    d["prev_act"], d["ttc"], frac, p, radar_variant=radar)
    assert bits(pp, inp["prev_err"])  # pos_error_prev: the value pos_error held on entry, bit for bit
    scale = d["target"].norm(dim=1) + d["pos"].norm(dim=1)
    compare(entry, "pos_error", pe, err, EPS * scale.unsqueeze(1))
    dist, vn = err.norm(dim=1), d["vlv"].norm(dim=1)
    dd, dvn = EPS * (scale + dist), EPS * vn
    dy = EPS * (d["target_yaw"].abs() + d["euler"][:, 2].abs() + 4 * math.pi)
    vdc = (d["vlv"] / (vn.unsqueeze(1) + 1e-6) * err / (dist.unsqueeze(1) + 1e-6)).sum(1)
    dvdc = 4 * EPS + dd / (dist + 1e-6)
    mult, k = 1 + 2 * frac, abs(p["vel_direction_component_reward_magnitude"])
    nm = L.LIDAR_NAV_PARAM_NAMES
    t_terms = (EPS * abs(p[nm[0]]) + slope(p[nm[0]], p[nm[1]]) * dd
               + EPS * abs(p[nm[2]]) + slope(p[nm[2]], p[nm[3]]) * dd + abs(p[nm[2]]) * (-p[nm[3]] * dist ** 2).exp() * slope(1, 2) * dy
               + k * (dvdc + slope(2, 2) * dvn + EPS) + (k + 0.2) * dd / 3
               + dd / 20 + EPS * (1 + dist / 20)
               + (slope(2, 2) * dvn + 2 * slope(2, 8) * EPS * d["vlv"][:, 0].abs() + 2 * slope(1, 2) * dd + EPS * 4)
               + (dist < 1 + dd) * ((slope(1.5, 10) + slope(1.5, 0.5)) * dvn + (slope(2, 0.2) + slope(4, 15) + 1.5 * slope(1, 2)) * dy
                                    + slope(1.5, 5) * EPS * d["bav"][:, 2].abs() + EPS * 9.5)  # stable: 0 unless dist < 1
               + 3 * EPS + 3 * math.sqrt(4 / math.e) * EPS * d["ttc"] ** 2)
    ab = (d["act"].abs() + d["prev_act"].abs())
    pens = sum(EPS * abs(p[nm[i]]) + slope(p[nm[i]], p[nm[i + 1]]) * EPS * ab[:, (i - 5) // 2 % 4] for i in range(5, 21, 2))
    tol = mult * (t_terms + pens) + EPS * ref.abs()
    # branch choices inside the reward: stable (dist < 1) and vdc > 0; within their bands either side is accepted
    # position 0 in an identity frame (the dist_1 / dist_3 / vdc_0 / tiny-speed constructions): err == target and vdc are exact in
    # float32 too, so those rows take the reference's side of both decisions
    exact = (d["pos"].abs().sum(1) == 0) & (d["veh"][:, 3] == 1)
    near_stable = ((dist - 1).abs() <= dd) & ~inp["crashes"] & ~exact
    near_vdc = (vdc.abs() <= dvdc) & (vn > 0) & ~inp["crashes"] & ~exact
    _exempt(entry, "stable", near_stable)
    _exempt(entry, "vdc_sign", near_vdc)
    tol = torch.where(near_stable | near_vdc, torch.full_like(tol, 1e9), tol)
    compare(entry, "reward", rew, ref, tol)
    assert bool((rew[inp["crashes"]] == float(np.float32(p["collision_penalty"]))).all())
    if N >= 129:
        rew2, pe2, _ = run(-inp["veh"])
        assert same(rew2, rew) and same(pe2, pe)
        _cover(entry, "q_neg")


@pytest.mark.parametrize("N", NS)
def test_lidar_nav_obs(N):
    entry = "lnav_obs"
    inp, g = _lnav_inputs(N, 500 + N)
    rows = _edge_rows(N, ["angle_0", "angle_2pi_pm_ulp", "angle_pm_pi", "dist_0", "q_neg"], N + 4)
    _angle_edges(inp, rows, "euler", (0, 1, 2))
    if "dist_0" in rows:
        inp["target"][rows["dist_0"]] = inp["pos"][rows["dist_0"]]
        inp["u_vec"][rows["dist_0"][::2]] = 0.5
    if "q_neg" in rows:
        inp["veh"][rows["q_neg"]] *= -1
    L_ = 24 + N % 3
    lidar = torch.rand(N, L_, generator=g) * 5
    null = N in (128, 4097)
    obs_stride = 17 + L_ + 5
    _cover(entry, *rows.keys(), *(["lidar_null"] if null else []), *(["obs_pad"] if obs_stride > 17 + L_ else []))
    if N % ENV_THREADS:
        _cover(entry, "ragged")
    stride = _stride(N)
    st = _state(N, stride, torch.Generator().manual_seed(N), pos=inp["pos"])

    def run(veh):
        lib = _lib.load()
        obs = torch.full((N, obs_stride), SENTINEL, device=DEV)
        t = [_dev(x) for x in (st, veh, inp["euler"], inp["blv"], inp["bav"], inp["act"], inp["target"], inp["target_yaw"], inp["u_vec"],
                               inp["u_euler"], lidar)]
        _lib.check(lib.agx_lidar_nav_obs(N, _p(t[0]), stride, *[_p(x) for x in t[1:10]], None if null else _p(t[10]), L_, _p(obs), obs_stride,
                                         None), "agx_lidar_nav_obs")
        torch.cuda.synchronize()
        return obs.cpu()

    obs = run(inp["veh"])
    d = {k: v.double() for k, v in inp.items() if v.is_floating_point()}
    ref = L.process_obs(d["veh"], d["pos"], d["target"], d["euler"], d["target_yaw"], d["blv"], d["bav"], d["act"], lidar.double(), d["u_vec"],
                        d["u_euler"])
    vec = O.quat_rotate_inverse(d["veh"], d["target"] - d["pos"])
    dist = vec.norm(dim=1)
    dv = EPS * (d["target"].norm(dim=1) + d["pos"].norm(dim=1) + dist)
    t_dir = (dv + EPS * 0.2) / dist + ref[:, 0:3].abs().amax(dim=1) * (dv / dist + EPS)
    compare(entry, "dir", obs[:, 0:3], ref[:, 0:3], t_dir.unsqueeze(1))
    compare(entry, "dist", obs[:, 3], ref[:, 3], dv)
    a = d["euler"][:, 0:2]
    wrap = ssa_wrap_near(O.ssa(a)).any(dim=1)
    compare(entry, "angles", obs[:, 4:6], ref[:, 4:6], EPS * (a.abs() + 2 * math.pi + 0.1), wrap=wrap)
    wrap6 = ssa_wrap_near(ref[:, 6])
    compare(entry, "yaw_error", obs[:, 6], ref[:, 6], EPS * (d["target_yaw"].abs() + d["euler"][:, 2].abs() + 4 * math.pi), wrap=wrap6)
    _exempt(entry, "ssa_wrap", wrap | wrap6)
    assert bits(obs[:, 7:17], torch.cat([inp["blv"], inp["bav"], inp["act"]], 1))
    if null:
        assert bool((obs[:, 17:] == SENTINEL).all())
    else:
        assert bits(obs[:, 17:17 + L_], lidar) and bool((obs[:, 17 + L_:] == SENTINEL).all())
    if N >= 129:
        assert same(run(-inp["veh"]), obs)
        _cover(entry, "q_neg")


# ---- motor-command position tasks (e2e_task.cu) and setpoint sim2real tasks (sim2real.cu) -----------------------------------------
def _pose_inputs(N, seed, stride):
    """state with position, a unit quaternion and a world velocity; edge rows of the quaternion applied by the callers"""
    g = torch.Generator().manual_seed(seed)
    st = _state(N, stride, g, pos=torch.randn(N, 3, generator=g) * 3, vel=torch.randn(N, 3, generator=g))
    return st, g


def _quat_edges(st, rows):
    """qw_0 / qw_neg0 / pitch_lock / angle edges of roll and yaw (built in float64, rounded once to float32) / q_neg"""
    pi = math.pi
    two = float(_ulps(F32_2PI, -1)), float(_ulps(F32_2PI, 1))
    if "qw_0" in rows:
        st[rows["qw_0"], 3:7] = f32([0.6, 0.0, -0.8, 0.0])
    if "qw_neg0" in rows:
        st[rows["qw_neg0"], 3:7] = f32([0.0, 0.6, 0.8, -0.0])
    if "pitch_lock" in rows:
        r = rows["pitch_lock"]
        k = torch.arange(len(r), dtype=torch.float64)
        p = (pi / 2 - 1e-4 * (k % 5) / 4) * torch.where(k % 2 == 0, 1.0, -1.0)
        st[r, 3:7] = _quat_from_euler64(0.3 * k, p, 1.0 - 0.2 * k)
    for name, ang in (("angle_0", [0.0, -1e-9]), ("angle_2pi_pm_ulp", list(two)), ("angle_pm_pi", [pi, -pi, float(np.float32(pi))])):
        if name in rows:
            r = rows[name]
            a = torch.tensor([ang[i % len(ang)] for i in range(len(r))], dtype=torch.float64)
            st[r, 3:7] = _quat_from_euler64(torch.where(torch.arange(len(r)) % 2 == 0, a, 0.1), torch.full_like(a, 0.2), a)
    if "q_neg" in rows:
        st[rows["q_neg"], 3:7] *= -1


def _e2e_params(tag, crash_dist):
    p = _lib.AgxE2ERewardParams()
    for k, v in E.E2E_PARAMS[tag].items():
        setattr(p, k, float(v))
    p.crash_dist = float(crash_dist)
    return p, {k: float(getattr(p, k)) for k in E.E2E_PARAMS[tag]}  # the float32 values the kernel receives


@pytest.mark.parametrize("N", NS)
def test_e2e_reward(N):
    entry, tag = "e2e_reward", ("end_to_end", "px4")[N % 2]
    stride = _stride(N)
    st, g = _pose_inputs(N, 600 + N, stride)
    tnull = N in (127, 4097)
    target = torch.zeros(N, 3) if tnull else st[:, 0:3] + torch.randn(N, 3, generator=g) * torch.rand(N, 1, generator=g) * 3
    prev = (target - st[:, 0:3]) + 0.05 * torch.randn(N, 3, generator=g)
    w = torch.randn(N, 3, generator=g)
    act, prev_act = torch.rand(N, 4, generator=g) + 0.2, torch.rand(N, 4, generator=g) + 0.2
    crashes = torch.rand(N, generator=g) < 0.03
    cd = 1.5
    names = ["dist_0", "dist_at_crash", "dist_eq_prev", "exp_underflow", "qw_0", "q_neg", "crash_in"]
    rows = _edge_rows(N, names, N + 5)
    _quat_edges(st, rows)
    if "dist_0" in rows:
        target[rows["dist_0"]] = st[rows["dist_0"], 0:3]
    if "dist_at_crash" in rows:  # position 0, axis-aligned target: dist == |target| exactly, at crash_dist and 1 ulp either side
        r = rows["dist_at_crash"]
        st[r, 0:3] = 0.0
        target[r] = f32([[cd, 0, 0], [0, float(_ulps(cd, 1)), 0], [0, 0, float(_ulps(cd, -1))]]).repeat(len(r), 1)[:len(r)]
    if "dist_eq_prev" in rows:
        prev[rows["dist_eq_prev"]] = target[rows["dist_eq_prev"]] - st[rows["dist_eq_prev"], 0:3]
    if "exp_underflow" in rows:
        r = rows["exp_underflow"]
        st[r, 7:10], w[r], act[r] = 300.0, -300.0, 1e3
    if "crash_in" in rows:
        crashes[rows["crash_in"]] = True
    if tnull:
        target.zero_()  # what the kernel reads for target_position == NULL
    _cover(entry, *rows.keys(), *(["target_null"] if tnull else []))
    if N % ENV_THREADS:
        _cover(entry, "ragged")
    params, p = _e2e_params(tag, cd)

    def run(state):
        lib = _lib.load()
        cr, rew = _dev(crashes.to(torch.uint8)), torch.full((N,), SENTINEL, device=DEV)
        t = [_dev(x) for x in (state, w, target, act, prev_act, prev)]
        _lib.check(lib.agx_e2e_reward(N, _p(t[0]), stride, _p(t[1]), None if tnull else _p(t[2]), _p(t[3]), _p(t[4]), _p(t[5]), C.byref(params),
                                      _p(cr), _p(rew), None), "agx_e2e_reward")
        torch.cuda.synchronize()
        return rew.cpu(), cr.cpu().bool()

    rew, cr = run(st)
    D = lambda t: t.double()
    x, q, v = D(st[:, 0:3]), D(st[:, 3:7]), D(st[:, 7:10])
    ref, ref_cr = E.compute_reward(D(target) - x, q, v, D(w), crashes, D(act), D(prev_act), D(prev), cd, p)
    dist, pd = (D(target) - x).norm(dim=1), D(prev).norm(dim=1)
    dd = EPS * (D(target).norm(dim=1) + x.norm(dim=1) + dist)
    decision(entry, "crash", cr, ref_cr, ((dist - cd).abs() <= dd) & ~crashes & (x.abs().sum(1) != 0))
    gains = max(p["towards_gain_pos"], p["towards_gain_neg"])
    P = 36.0
    dpe = dd * (p["z_error_scale"] + 2) * (slope(10, 10) + slope(2, 2))
    aux = (p["align_gain1"] + p["align_gain2"] + 3 + 3 * p["angvel_gain"] + 4 * p["action_diff_gain"] + 2.5 + p["upright_gain2"] + 0.04)
    dterms = (EPS * 4 * (slope(2.5, 5) + slope(p["upright_gain2"], p["upright_exp2"]) + slope(p["align_gain1"], p["align_exp1"])
                         + slope(p["align_gain2"], p["align_exp2"]))
              + slope(p["angvel_gain"], 10) * EPS * D(w).abs().sum(1) + slope(1, 5) * EPS * v.abs().sum(1)
              + slope(0.01, 10) * EPS * (D(act).abs() + p["hover_thrust"]).sum(1)
              + slope(p["action_diff_gain"], 6) * EPS * (D(act).abs() + D(prev_act).abs()).sum(1) + EPS * aux)
    tol = gains * (dd + EPS * (dist + pd)) + ((dpe + EPS * P) * (1 + aux) + P * dterms + dterms) / 100 + EPS * ref.abs()
    compare(entry, "reward", rew, ref, tol)
    if N >= 129:
        s2 = st.clone()
        s2[:, 3:7] *= -1
        r2, c2 = run(s2)
        assert same(r2, rew) and torch.equal(c2, cr)
        _cover(entry, "q_neg")


@pytest.mark.parametrize("N", NS)
def test_e2e_obs(N):
    entry = "e2e_obs"
    stride = _stride(N)
    st, g = _pose_inputs(N, 700 + N, stride)
    tnull = N in (128, 65537)
    target = torch.zeros(N, 3) if tnull else torch.randn(N, 3, generator=g) * 3
    w, noise = torch.randn(N, 3, generator=g), torch.randn(N, 12, generator=g) * 0.01
    rows = _edge_rows(N, ["pitch_lock", "qw_0", "angle_pm_pi", "q_neg"], N + 6)
    _quat_edges(st, rows)
    obs_stride = 15 + 1 + N % 4
    _cover(entry, *rows.keys(), *(["obs_pad"] if obs_stride > 15 else []), *(["target_null"] if tnull else []))
    if N % ENV_THREADS:
        _cover(entry, "ragged")

    def run(state):
        lib = _lib.load()
        obs = torch.full((N, obs_stride), SENTINEL, device=DEV)
        t = [_dev(x) for x in (state, w, target, noise)]
        _lib.check(lib.agx_e2e_obs(N, _p(t[0]), stride, _p(t[1]), None if tnull else _p(t[2]), _p(t[3]), _p(obs), obs_stride, None), "agx_e2e_obs")
        torch.cuda.synchronize()
        return obs.cpu()

    obs = run(st)
    D = lambda t: t.double()
    x, q = D(st[:, 0:3]), D(st[:, 3:7])
    ref = E.process_obs(x, q, D(st[:, 7:10]), D(w), D(target), D(noise))
    compare(entry, "pos", obs[:, 0:3], ref[:, 0:3], EPS * (D(target).abs() + x.abs() + D(noise[:, 0:3]).abs()))
    R = E.quaternion_to_matrix(q[:, [3, 0, 1, 2]])
    cp = torch.hypot(R[:, 0, 0], R[:, 1, 0])
    s = R[:, 2, 0].abs().clamp(max=1)
    d_ang = 2 * (4 * EPS / cp) + torch.minimum(2 * EPS / (1 - s * s).clamp(min=1e-300).sqrt(), torch.full_like(s, math.sqrt(4 * EPS)))
    # the reference's own float32 arithmetic (pytorch3d's) takes asin of R20 unclamped: where float32 |R20| rounds past 1 it is nan too
    R32 = E.quaternion_to_matrix(st[:, [6, 3, 4, 5]])
    dom = R32[:, 2, 0].abs() > 1
    _exempt(entry, "asin_domain", dom)
    got6 = torch.where(dom.unsqueeze(1) & obs[:, 3:9].isnan(), ref[:, 3:9].float(), obs[:, 3:9])
    compare(entry, "rot6d", got6, ref[:, 3:9], (2 * d_ang + 6 * EPS).unsqueeze(1))
    assert bits(obs[:, 9:15], (D(torch.cat([st[:, 7:10], w], 1)) + D(noise[:, 6:12])).float())  # one rounding: float32 of the exact sum
    assert bool((obs[:, 15:] == SENTINEL).all())
    if N >= 129:
        s2 = st.clone()
        s2[:, 3:7] *= -1
        assert same(run(s2), obs)
        _cover(entry, "q_neg")


def _euler_cond(q):
    """float64 (roll, pitch, yaw) error bounds of euler_xyz_0_2pi + ssa on q: atan2 over hypot of its arguments, asin near +-1"""
    qx, qy, qz, qw = q.unbind(1)
    hr = torch.hypot(2 * (qw * qx + qy * qz), qw * qw - qx * qx - qy * qy + qz * qz)
    hy = torch.hypot(2 * (qw * qz + qx * qy), qw * qw + qx * qx - qy * qy - qz * qz)
    s = (2 * (qw * qy - qz * qx)).abs().clamp(max=1)
    dp = torch.minimum(4 * EPS / (1 - s * s).clamp(min=1e-300).sqrt(), torch.full_like(s, math.sqrt(8 * EPS)))
    return 4 * EPS / hr + 4 * math.pi * EPS, dp + 4 * math.pi * EPS, 4 * EPS / hy + 4 * math.pi * EPS


@pytest.mark.parametrize("variant", [0, 1])
@pytest.mark.parametrize("N", NS)
def test_s2r_reward(N, variant):
    entry = "s2r_reward"
    stride = _stride(N)
    st, g = _pose_inputs(N, 800 + N + variant, stride)
    tnull, aout_null = N in (128, 4097), variant == 1 and N in (127, 65537)
    target = st[:, 0:3] + torch.randn(N, 3, generator=g) * torch.rand(N, 1, generator=g) * 12
    veh = _quat_from_euler64(torch.zeros(N), torch.zeros(N), torch.rand(N, generator=g, dtype=torch.float64) * 2 * math.pi)
    blv = torch.randn(N, 3, generator=g)
    act, prev_act = torch.rand(N, 4, generator=g) * 2 - 1, torch.rand(N, 4, generator=g) * 2 - 1
    crashes = torch.rand(N, generator=g) < 0.03
    names = ["dist_10_pm_ulp", "dist_eq_prev", "dist_0", "angle_0", "angle_2pi_pm_ulp", "angle_pm_pi", "pitch_lock", "qw_0", "crash_in", "q_neg"]
    rows = _edge_rows(N, names, N + 7 + variant)
    _quat_edges(st, rows)
    if tnull:
        target.zero_()
    prev_dist = ((target - st[:, 0:3]).norm(dim=1) + torch.randn(N, generator=g) * 0.05).abs()
    for name in ("dist_10_pm_ulp", "dist_eq_prev"):
        if name in rows:  # position 0, identity frames, axis-aligned target: dist == |target| exactly
            r = rows[name]
            st[r, 0:3], st[r, 3:7], veh[r] = 0.0, f32([0, 0, 0, 1]), f32([0, 0, 0, 1])
            if not tnull:
                x = [10.0, float(_ulps(10.0, 1)), float(_ulps(10.0, -1)), float(_ulps(10.0, 3))] if name == "dist_10_pm_ulp" else [2.5, 7.0]
                target[r] = torch.stack([torch.tensor([0.0, x[i % len(x)], 0.0]) for i in range(len(r))])
            prev_dist[r] = target[r].norm(dim=1) if name == "dist_eq_prev" else prev_dist[r]
    if "dist_0" in rows:
        st[rows["dist_0"], 0:3] = target[rows["dist_0"]]
    if "crash_in" in rows:
        crashes[rows["crash_in"]] = True
    _cover(entry, *rows.keys(), *(["target_null"] if tnull else []), *(["act_out_null"] if aout_null else []))
    if N % ENV_THREADS:
        _cover(entry, "ragged")

    def run(state, vq):
        lib = _lib.load()
        cr, rew, av = _dev(crashes.to(torch.uint8)), torch.full((N,), SENTINEL, device=DEV), torch.full((N, 4), SENTINEL, device=DEV)
        t = [_dev(x) for x in (state, vq, blv, target, prev_dist, act, prev_act)]
        _lib.check(lib.agx_s2r_reward(N, variant, _p(t[0]), stride, _p(t[1]), _p(t[2]), None if tnull else _p(t[3]), _p(t[4]), _p(t[5]), _p(t[6]),
                                      None if aout_null else _p(av), _p(cr), _p(rew), None), "agx_s2r_reward")
        torch.cuda.synchronize()
        return rew.cpu(), cr.cpu().bool(), av.cpu()

    rew, cr, av = run(st, veh)
    D = lambda t: t.double()
    x, q = D(st[:, 0:3]), D(st[:, 3:7])
    ref, ref_cr, ref_act = S.reward(variant, x, q, D(veh), D(blv), D(target), D(prev_dist), D(act), D(prev_act), crashes)
    d = D(target) - x
    dist, pd = S._quat_apply_inverse(q if variant else D(veh), d).norm(dim=1), D(prev_dist)
    dd = EPS * (D(target).norm(dim=1) + x.norm(dim=1) + dist)
    exact = (x.abs().sum(1) == 0) & ((q[:, 3] == 1) if variant else (D(veh)[:, 3] == 1))  # the axis-aligned constructions: exact
    near_crash = ((dist - 10).abs() <= dd) & ~crashes & ~exact
    decision(entry, "crash", cr, ref_cr, near_crash)
    _exempt(entry, "closer_side", ((dist - pd).abs() <= dd) & ~exact)  # dist < prev_dist: either gain times a difference within the bar
    _, _, dyaw = _euler_cond(q)
    gain = 1200.0 if variant else 400.0
    dcl = gain * (dd + EPS * (dist + pd))
    P = 8.0
    dP = EPS * 8 + (4 * dist * (-dist ** 2).exp() + 60 * dist * (-10 * dist ** 2).exp() + 150 * (-50 * dist).exp()) * dd  # |dP/ddist| dd
    cl = (1200.0 if variant else 400.0) * (pd - dist).abs()
    da = EPS * (3 * D(act).abs().sum(1) + 1)
    dap = 4 * 0.3 * da + EPS * 1.2
    dadp = 6 * 0.4 * (da + EPS * D(prev_act).abs().sum(1)) + EPS * 1.6
    dsp = (slope(2, 2.5) + slope(1, 3)) * EPS * D(blv).norm(dim=1) + EPS * 2
    dyr = 15 * dyaw + EPS * 3
    big = ref.abs() + P * (4 + cl) + cl + 10
    tol = dP * (3 + cl / 9) + P * (dcl / 9 + dap + dsp) + dd / 40 + dap + dadp + dcl + dyr + dsp + EPS * big
    tol = torch.where(near_crash, torch.full_like(tol, 1e9), tol)
    compare(entry, "reward", rew, ref, tol)
    assert bool((rew[cr] == -50.0).all())
    if variant and not aout_null:
        compare(entry, "act_vehicle", av[:, 0:3], ref_act[:, 0:3], (3 * EPS * D(act[:, 0:3]).abs().sum(1)).unsqueeze(1))
        assert bits(av[:, 3], act[:, 3])
    else:
        assert bool((av == SENTINEL).all())  # actions_vehicle_frame untouched (velocity variant, or NULL)
    if N >= 129:
        s2 = st.clone()
        s2[:, 3:7] *= -1
        r2, c2, a2 = run(s2, -veh)
        assert same(r2, rew) and torch.equal(c2, cr) and same(a2, av)
        _cover(entry, "q_neg")


@pytest.mark.parametrize("N", NS)
def test_s2r_obs(N):
    entry = "s2r_obs"
    stride = _stride(N)
    st, g = _pose_inputs(N, 900 + N, stride)
    tnull = N in (1, 129, 65537)
    target = torch.zeros(N, 3) if tnull else torch.randn(N, 3, generator=g) * 3
    blv, bav, act, noise = (torch.randn(N, 3, generator=g), torch.randn(N, 3, generator=g), torch.rand(N, 4, generator=g) * 2 - 1,
                            torch.randn(N, 12, generator=g))
    rows = _edge_rows(N, ["qw_0", "qw_neg0", "q_neg", "angle_0", "angle_2pi_pm_ulp", "angle_pm_pi", "pitch_lock"], N + 8)
    _quat_edges(st, rows)
    obs_stride = 17 + 2 + N % 3
    _cover(entry, *rows.keys(), *(["obs_pad"] if obs_stride > 17 else []), *(["target_null"] if tnull else []))
    if N % ENV_THREADS:
        _cover(entry, "ragged")

    def run(state):
        lib = _lib.load()
        sd, obs = _dev(state), torch.full((N, obs_stride), SENTINEL, device=DEV)
        t = [_dev(x) for x in (blv, bav, act, target, noise)]
        _lib.check(lib.agx_s2r_obs(N, _p(sd), stride, _p(t[0]), _p(t[1]), _p(t[2]), None if tnull else _p(t[3]), _p(t[4]), _p(obs), obs_stride,
                                   None), "agx_s2r_obs")
        torch.cuda.synchronize()
        return obs.cpu(), sd.cpu()

    obs, st_after = run(st)
    D = lambda t: t.double()
    x, q = D(st[:, 0:3]), D(st[:, 3:7])
    ref, q_after = S.process_obs(x, q, D(blv), D(bav), D(act), D(target), D(noise))
    # in place: the quaternion times sign(qw) (0 at qw = +-0), bit for bit; every other state column keeps its bits
    assert bits(st_after[:, 3:7], q_after.float())
    assert bits(torch.cat([st_after[:, 0:3], st_after[:, 7:]], 1), torch.cat([st[:, 0:3], st[:, 7:]], 1))
    compare(entry, "pos", obs[:, 0:3], ref[:, 0:3], EPS * (D(target).abs() + x.abs() + 0.03 * D(noise[:, 3:6]).abs()))
    dr, dp, dy = _euler_cond(q_after)
    e = O.ssa(O.euler_xyz_from_quat(q_after))
    flip = ssa_wrap_near(e[:, 0]) | ssa_wrap_near(e[:, 2])  # roll or yaw at the wrap: the quaternion may come out negated
    _exempt(entry, "ssa_wrap", flip)
    compare(entry, "quat", obs[:, 3:7], ref[:, 3:7], (dr + dp + dy + 4 * EPS).unsqueeze(1), sign_flip=flip)
    compare(entry, "vel", obs[:, 7:13], ref[:, 7:13], EPS * (D(torch.cat([blv, bav], 1)).abs() + 0.02 * D(noise[:, 6:12]).abs()))
    assert bits(obs[:, 13:17], act) and bool((obs[:, 17:] == SENTINEL).all())
    if N >= 129:
        keep = st[:, 6] != 0  # at qw = +-0 the sign normalisation zeroes q, and the zeros' signs follow q's
        s2 = st.clone()
        s2[:, 3:7] *= -1
        o2, a2 = run(s2)
        assert same(o2[keep], obs[keep]) and same(a2[keep, 3:7], st_after[keep, 3:7])
        _cover(entry, "q_neg")


# ---- argument validation not covered elsewhere -------------------------------------------------------------------------------------
def test_argument_validation():
    lib = _lib.load()
    x = torch.zeros(64, device=DEV)
    args = lambda W: (1, 1, W, 1, 1, _p(x), _p(x), 13, 10.0, 0.2, 10.0, 10.0, _p(x), _p(x), None)
    assert lib.agx_lidar_nav_pool(*args(2134)) == -1  # 2134 x 12 B per band x 8 warps > 200 KB
    msg = lib.agx_last_error()
    assert b"shared memory" in msg and b"25608 B x 8 warps" in msg, msg
    o, a = torch.zeros(4, 40, device=DEV), torch.zeros(4, 4, device=DEV)
    nav = lambda lidar, L_, stride: lib.agx_lidar_nav_obs(1, _p(x), 13, *[_p(x)] * 4, _p(a), *[_p(x)] * 4, lidar, L_, _p(o), stride, None)
    assert nav(_p(x), 20, 36) == -1 and b"stride too small" in lib.agx_last_error()  # obs_stride < 17 + num_lidar
    assert nav(None, 20, 17) != -1  # lidar_obs == NULL: num_lidar is ignored
    assert lib.agx_lidar_nav_obs(1, _p(x), 13, *[_p(x)] * 4, _p(a), *[_p(x)] * 4, _p(x), -1, _p(o), 40, None) == -1


# ---- runs last (file order) --------------------------------------------------------------------------------------------------------
def test_zz_exemptions_are_rare_and_every_edge_ran(request):
    tests = [f for n, f in globals().items() if n.startswith("test_") and f is not test_zz_exemptions_are_rare_and_every_edge_ran]
    expected = sum(math.prod(len(m.args[1]) for m in getattr(f, "pytestmark", []) if m.name == "parametrize") for f in tests)
    if len(DONE) < expected:
        pytest.skip(f"{len(DONE)} of the module's {expected} other tests ran: coverage and exemption rates need all of them")
    missing = sorted((e, k) for e, ks in EDGES.items() for k in ks if (e, k) not in COVER)
    assert not missing, missing
    for (entry, what), (n, total) in sorted(EXEMPT.items()):
        assert n <= max(1, 0.01 * total), (entry, what, n, total)
