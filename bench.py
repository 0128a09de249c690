#!/usr/bin/env python
"""bench.py -- env-steps/sec of the position_setpoint_task hot path (BASELINE.json configs[1]).

    python bench.py --gpus 1 --steps 200 --warmup 10            # our arm (CUDA, C ABI)
    python bench.py --impl reference --steps 20 --warmup 3      # reference arm (CPU, see below)
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 \
           --master-port P bench.py --gpus N --steps K --warmup W

One "step" = one PositionSetpointTask.step over one batch of 65,536 envs per GPU (weak scaling:
per-GPU work fixed): fused physics + reward + termination/truncation + in-kernel reset +
observation and (N > 1) the all-gather of the observation tensor: hand-written NVLink push / wait
kernels that run BESIDE the chained step launches on a side stream (the push of step t overlaps step
t+1; the K-th gather has landed on every rank before the closing event; --gather sync|nccl for the
per-step-awaited and the NCCL variants).  The step of an 8-GPU run must RECEIVE 7 x 3.4 MB of rows:
`roofline.nvlink_floor_us` = that ingress / 450 GB/s (H100 NVLink, one direction) is the floor of the step period at N > 1.

Timing: W >= 3 warm-up steps, then exactly K steps bracketed by barrier + synchronize and one
CUDA-event pair on the launching stream.  One 65,536-env working set (~12 MB) fits in the H100's
50 MB L2, so the timed loop rotates over R = 16 independent replicas of the environment batch
(~190 MB of state in total, several times L2): every step finds its state cold in L2, nothing is
flushed and no step is skipped.  value = N_gpus * envs * K / elapsed, max over ranks.
`value_hot_l2` is the same loop on a single replica (state resident in L2; every tile's step waits for
that tile's previous step -- the dependent-chain figure, what a policy-free rollout of ONE batch sees).
Step launches are chained per 32-env tile, not per grid (hp1.cu "chained steps"), so in the rotating
loop the tail of one replica's step overlaps the next replica's step.

Sub-lines of the same JSON line at N = 1: `hp2_depth` (north_star's 64x48 depth target), `config3_*` / `config4_*` / `config5_env_sweep`
(BASELINE configs[2..4] at full size) and `navigation_task_e2e`.  They are single-GPU workloads: at N > 1 they are skipped unless
--multi-gpu-sublines is given (the N > 1 line is the headline workload with its all-gather, and the sharded-task e2e).

Reference arm (`--impl reference`): the reference's Isaac Gym sim_device=cpu pipeline cannot run
here or on the GPU box (isaacgym is a closed binary, not installed).  What CAN run is the reference's
own torch control stack: `__graft_entry__.build()` installs the unmodified reference into the
git-ignored `baseline/_ref` (pip --no-deps; it travels with the snapshot) and oracle/reference_arm.py
drives its BaseMultirotor.step / compute_reward / reset_idx on the host cores, with the oracle's
rigid-body integrator standing in for PhysX (`kind: "reference"`).  Where baseline/_ref is missing
the oracle port of the same step is timed instead (`kind: "port"`).  Rank 0 runs it with every host
thread, whatever --gpus says (torchrun's OMP_NUM_THREADS=1 is overridden).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

ENVS_PER_GPU = 65536
ALG_BYTES_PER_ENV_STEP = 210  # SURVEY.md section 8(d): 84 B read + 126 B written, state-only, M = 4
METRIC = "env-steps/sec (position_setpoint_task, base_quadrotor, lee_attitude_control, 65536 envs/GPU, state-only)"


def workload_config(n_gpus, extra=None):
    cfg = {
        "workload": "position_setpoint_task/base_quadrotor/lee_attitude_control/empty_env",
        "envs_per_gpu": ENVS_PER_GPU,
        "global_envs": ENVS_PER_GPU * n_gpus,
        "physics_steps_per_env_step": 1,
        "dt": 0.01,
        "episode_len_steps": 500,
        "actions": "U(-1,1) resampled from 8 pre-generated batches",
        "parallelism": f"env-sharded x{n_gpus}" + (" + all-gather(obs) every step" if n_gpus > 1 else ""),
        "l2": "inputs larger than L2: timed loop rotates over 16 replicas of the env batch (~190 MB); consecutive step "
              "launches are chained per 32-env tile (programmatic dependent launch), so steps of different replicas overlap "
              "in flight; value_hot_l2 = one replica stepped back to back (every step waits for its own previous step)",
    }
    if extra:
        cfg.update(extra)
    return cfg


# ------------------------------------------------------------------------------------------
# clocks sampler
# ------------------------------------------------------------------------------------------
class ClockSampler:
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,"
         "clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index=0):
        self.rows, self.proc, self.gpu = [], None, gpu_index

    def start(self):
        try:
            self.proc = subprocess.Popen(
                ["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-lms", "50", "-i", str(self.gpu)],
                stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([x.strip() for x in line.split(",")])

    def stop(self):
        if not self.proc:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        try:
            self.proc.wait(timeout=2)
        except Exception:
            pass
        sm, mx, reasons = [], None, set()
        for r in self.rows:
            try:
                sm.append(float(r[1]))
                mx = float(r[2])
                for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), r[5:9]):
                    if v.lower().startswith("active"):
                        reasons.add(name)
            except (ValueError, IndexError):
                continue
        # "under load" = samples in the top half of the observed clock range
        load = [x for x in sm if x >= 0.5 * max(sm)] if sm else []
        return {"sm_mhz": statistics.median(load) if load else None, "sm_max_mhz": mx, "samples": len(sm),
                "reasons": sorted(reasons)}


# ------------------------------------------------------------------------------------------
# CPU port (oracle) timing -- cpu_baseline leg and the reference arm
# ------------------------------------------------------------------------------------------
def time_cpu_port(n_envs, steps, warmup):
    import torch

    from oracle import hp1_oracle as O

    model = O.Hp1Model()
    g = torch.Generator().manual_seed(0)
    st = O.make_state(model, n_envs)
    O.reset_envs(model, st, torch.ones(n_envs, dtype=torch.bool), O.draw_reset_uniforms(model, n_envs, generator=g))
    st.sim_steps = (torch.arange(n_envs) % 500).to(torch.int32)
    tgt = torch.zeros(n_envs, 3)
    acts = [torch.rand(n_envs, 4, generator=g) * 2 - 1 for _ in range(8)]
    draw = lambda: O.draw_reset_uniforms(model, n_envs, generator=g)
    for i in range(warmup):
        O.position_task_step(model, st, acts[i % 8], tgt, draw_fn=draw)
    # torch's CPU ops do not scale to every core for [N,3]-sized tensors: use the fastest of a few
    # thread counts (so the baseline is the best the host can do, and `cores` is what was used)
    max_t = torch.get_num_threads()
    best = (None, float("inf"))
    for nt in sorted({max_t, max(1, max_t // 2), max(1, max_t // 4), min(max_t, 8)}, reverse=True):
        torch.set_num_threads(nt)
        O.position_task_step(model, st, acts[0], tgt, draw_fn=draw)
        t0 = time.perf_counter()
        for i in range(2):
            O.position_task_step(model, st, acts[i % 8], tgt, draw_fn=draw)
        dt_ = time.perf_counter() - t0
        if dt_ < best[1]:
            best = (nt, dt_)
    torch.set_num_threads(best[0])
    t0 = time.perf_counter()
    for i in range(steps):
        O.position_task_step(model, st, acts[i % 8], tgt, draw_fn=draw)
    dt = time.perf_counter() - t0
    used = torch.get_num_threads()
    torch.set_num_threads(max_t)
    return n_envs * steps / dt, dt / steps, used


def host_threads():
    """threads this process may use: torchrun exports OMP_NUM_THREADS=1 to every rank, which is not the host's capacity"""
    try:
        return max(1, len(os.sched_getaffinity(0)))
    except AttributeError:
        return max(1, os.cpu_count() or 1)


def time_cpu_reference(n_envs, steps, warmup):
    """(value, s/step, threads, kind, note): the reference's own control stack from baseline/_ref when it was staged
    (oracle/reference_arm.py), else the oracle port"""
    import torch

    torch.set_num_threads(host_threads())
    from oracle import reference_arm as RA

    if RA.staged():
        # the reference logs to stdout (its own logger and a print in control_allocation.py): keep stdout to the one JSON line
        sys.stdout.flush()
        saved = os.dup(1)
        os.dup2(2, 1)
        try:
            v, per, cores = RA.time_reference(n_envs, steps, warmup)
        finally:
            sys.stdout.flush()
            os.dup2(saved, 1)
            os.close(saved)
        return v, per, cores, "reference", ("unmodified reference control stack (baseline/_ref: BaseMultirotor.step, compute_reward, reset_idx) on torch CPU + "
                                            "the oracle's rigid-body integrator in place of PhysX (closed binary, not installable); NOT the Isaac Gym CPU pipeline")
    v, per, cores = time_cpu_port(n_envs, steps, warmup)
    return v, per, cores, "port", "oracle port of the reference step (baseline/_ref was not staged on this box)"


def run_reference_arm(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return 0  # rank 0 alone measures the host: it uses every host thread, whatever the number of GPUs
    n_envs = ENVS_PER_GPU
    # bound the sample: keep the whole run within ~2 minutes of CPU time
    _, t1, _, _, _ = time_cpu_reference(n_envs, 1, 1)
    budget = 120.0
    if (args.steps + args.warmup) * t1 > budget:
        n_envs = max(1024, int(n_envs * budget / ((args.steps + args.warmup) * t1)) // 1024 * 1024)
    value, per_step, cores, kind, note = time_cpu_reference(n_envs, args.steps, max(args.warmup, 1))
    sample = f"{n_envs} envs x {args.steps} steps, torch CPU fp32, {cores} threads (of {host_threads()} available to the process)"
    line = {
        "impl": "reference", "metric": METRIC, "value": value, "unit": "env-steps/s", "n_gpus": args.gpus,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": per_step * 1e3, "higher_is_better": True,
        "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": workload_config(args.gpus, {"l2": "n/a (CPU)", "sample_envs": n_envs, "note": note + "; a host measurement: the same "
                                              "whole-host throughput is reported for every --gpus N (rank 0 runs it with all host threads)"}),
        "cpu_baseline": {"value": value, "unit": "env-steps/s", "cores": cores, "kind": kind, "sample": sample},
        "e2e": {"value": value, "unit": "env-steps/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0,
    }
    print(json.dumps(line))
    return 0


# ------------------------------------------------------------------------------------------
# our arm
# ------------------------------------------------------------------------------------------
def run_ours(args):
    import torch
    import torch.distributed as dist

    from aerial_gym_simulator_b200.distributed import ObsAllGather, PipelinedObsGather
    from aerial_gym_simulator_b200.hp1 import Hp1Engine, MultirotorSpec

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if world != args.gpus and world > 1:
        raise SystemExit(f"--gpus {args.gpus} but WORLD_SIZE={world}")
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    if world > 1:
        if os.environ.get("NCCL_DEBUG", "").upper() in ("", "VERSION"):
            os.environ["NCCL_DEBUG"] = "WARN"  # keep stdout to the single JSON line
        dist.init_process_group("nccl", device_id=dev)
    K, W = args.steps, max(args.warmup, 3)
    N = args.envs

    spec = MultirotorSpec()
    R = 16
    engines = []
    for rep in range(R):
        e = Hp1Engine(spec, N, dev, seed=1 + rep, env_id_offset=rank * N, device_rng_reset=True, strict_stale_obs=True,
                      materialize_derived=False)
        e.reset(torch.ones(N, dtype=torch.bool, device=dev))
        e.refresh()
        e.sim_steps.copy_((torch.arange(N, device=dev) % 500).int())  # de-synchronised episode phases
        engines.append(e)
    eng = engines[0]
    g = torch.Generator(device=dev).manual_seed(1234 + rank)
    acts = [(torch.rand(N, 4, generator=g, device=dev) * 2 - 1).contiguous() for _ in range(8)]
    gather, nccl_gather = None, None
    if world > 1:
        nccl_gather = ObsAllGather(N, 13, world * N, dev)  # the library collective: fallback and checker of the hand-written one
        if args.gather != "nccl":
            try:  # symmetric-memory rendezvous (NVLink peer mappings); every rank must take the same branch
                gather = PipelinedObsGather(N, 13, dev, num_buffers=4, max_ctas=args.gather_ctas)
                ok = torch.ones(1, device=dev)
            except Exception as exc:  # noqa: BLE001  -- e.g. a box without P2P between some GPU pair
                sys.stderr.write(f"[bench rank {rank}] {args.gather} gather unavailable ({exc!r})\n")
                gather, ok = None, torch.zeros(1, device=dev)
            dist.all_reduce(ok, op=dist.ReduceOp.MIN)
            if float(ok.item()) == 0.0:  # somebody failed: everybody uses the library collective, and the line says so
                args.gather, gather = "nccl", None
        if gather is not None:  # the push kernel of every step runs on the gather's side stream, beside the chained steps
            for e in engines:
                e.attach_obs_gather(gather)
    stream = torch.cuda.current_stream(dev)
    last = {"engine": eng}

    def step(i, mid=None, rotate=True, sync_gather=False):
        e = engines[i % R] if rotate else eng
        e.position_task_step(acts[i % 8], mid_event=mid)
        last["engine"] = e
        if world > 1:
            if gather is None:
                nccl_gather(e.obs)
            elif sync_gather or args.gather == "sync":
                gather.wait()  # this step's rows of every rank are here before the next step is launched

    def drain():
        """everything the steps enqueued so far -- pushes included -- is ordered before what follows on `stream`"""
        if gather is not None:
            gather.fence()
            gather.wait()

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize(dev)

    sampler = ClockSampler(local_rank)
    if rank == 0:
        sampler.start()  # samples across warm-up, the timed region and the follow-up loops
    for i in range(max(W, R)):  # every replica is stepped at least once before timing
        step(i)
    drain()
    barrier()
    if gather is not None:  # a bounded wait that expired during warm-up is reported where it happened (the words are sticky)
        w = int(gather.error_word.item())
        ew = [hex(int(e_.any_reset[2].item())) for e_ in engines if int(e_.any_reset[2].item())]
        if w or ew:
            sys.stderr.write(f"[bench rank {rank}] after warm-up: gather error word {hex(w)}, engine error words {ew[:4]}\n")

    # ---- timed region: exactly K steps over rotating replicas ------------------------------------
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    barrier()
    t_wall0 = time.perf_counter()
    ev0.record(stream)
    for i in range(K):
        step(i)
    drain()  # N > 1: the K-th gather has landed on this rank too, inside the timed region
    ev1.record(stream)
    t_enqueue = time.perf_counter() - t_wall0  # host time to enqueue the K steps (launches are asynchronous)
    barrier()
    t_wall = time.perf_counter() - t_wall0
    total_ms = torch.tensor([ev0.elapsed_time(ev1)], device=dev, dtype=torch.float64)
    if world > 1:
        dist.all_reduce(total_ms, op=dist.ReduceOp.MAX)
    total_s = float(total_ms.item()) * 1e-3
    value = world * N * K / total_s
    if args.dump_outputs and rank == 0:  # before the loops below step the same engines again
        dump_outputs(args.dump_outputs, last["engine"])

    # ---- N > 1: (a) self-check -- the gathered buffer of the last timed step equals the library collective's gather of the same
    # observation, on every rank; (b) the same loop with the gather awaited after EVERY step (what a policy in the loop sees) ----
    gather_check, value_sync = None, None
    if world > 1:
        e = last["engine"]
        if gather is not None:
            got = gather.wait().clone()
            want = nccl_gather(e.obs).clone()
            okc = torch.tensor([int(torch.equal(got, want))], device=dev)
            for chk in [gather.check] + [e_.check for e_ in engines]:
                try:
                    chk()
                except Exception as exc:  # noqa: BLE001
                    sys.stderr.write(f"[bench rank {rank}] {exc}\n")
                    okc.zero_()
            dist.all_reduce(okc, op=dist.ReduceOp.MIN)
            gather_check = bool(okc.item())
            for i in range(R):
                step(i, sync_gather=True)
            barrier()
            l0, l1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            l0.record(stream)
            for i in range(K):
                step(i, sync_gather=True)
            l1.record(stream)
            barrier()
            sync_ms = torch.tensor([l0.elapsed_time(l1)], device=dev, dtype=torch.float64)
            dist.all_reduce(sync_ms, op=dist.ReduceOp.MAX)
            value_sync = world * N * K / (float(sync_ms.item()) * 1e-3)

    # ---- dominant kernel alone: per-step event pairs.  At this size the fused step is ONE
    # launch (hp1_step_kernel<4,true,coop>), so the pair brackets exactly that kernel; on the
    # two-launch path the library would record the second event between main kernel and obs pass.
    Kk = min(K, 200)
    k0 = [torch.cuda.Event(enable_timing=True) for _ in range(Kk)]
    k1 = [torch.cuda.Event(enable_timing=True) for _ in range(Kk)]
    barrier()
    for i in range(Kk):
        e = engines[i % R]
        k0[i].record(stream)
        e.position_task_step(acts[i % 8])
        k1[i].record(stream)
    drain()
    barrier()
    main_total = torch.tensor([sum(a_.elapsed_time(b_) for a_, b_ in zip(k0, k1))], device=dev, dtype=torch.float64)
    if world > 1:
        dist.all_reduce(main_total, op=dist.ReduceOp.MAX)

    # ---- same loop, no flush (state L2-resident) ---------------------------------------------
    barrier()
    a0, a1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a0.record(stream)
    for i in range(K):
        step(i, rotate=False)
    drain()
    a1.record(stream)
    barrier()
    hot_ms = torch.tensor([a0.elapsed_time(a1)], device=dev, dtype=torch.float64)
    if world > 1:
        dist.all_reduce(hot_ms, op=dist.ReduceOp.MAX)
    value_hot = world * N * K / (float(hot_ms.item()) * 1e-3)

    # ---- the same rotating loop on engines configured like the task API's (EnvManager passes materialize_derived=True: the five
    # derived-state arrays of BaseMultirotor.update_states, 64 B/env, are written every step) -- N = 1 only, no gather ----------------
    value_api = None
    if world == 1:
        api_engines = []
        for rep in range(R):
            e = Hp1Engine(spec, N, dev, seed=1 + rep, env_id_offset=rank * N, device_rng_reset=True, strict_stale_obs=True, materialize_derived=True)
            e.reset(torch.ones(N, dtype=torch.bool, device=dev))
            e.refresh()
            e.sim_steps.copy_((torch.arange(N, device=dev) % 500).int())
            api_engines.append(e)
        for i in range(R):
            api_engines[i].position_task_step(acts[i % 8])
        barrier()
        b0, b1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        b0.record(stream)
        for i in range(K):
            api_engines[i % R].position_task_step(acts[i % 8])
        b1.record(stream)
        barrier()
        value_api = N * K / (b0.elapsed_time(b1) * 1e-3)
        del api_engines

    # ---- e2e: the call a user makes -- task_registry.make_task(...).step(actions) -- with HOST
    # buffers: pinned actions in, obs / reward / terminations / truncations out, every step ---------
    import aerial_gym_simulator_b200.task  # noqa: F401  (registers tasks)
    from aerial_gym_simulator_b200.registry.task_registry import task_registry

    tcfg = task_registry.get_task_config("position_setpoint_task")

    def make_task(host_io):
        old_args, old_dev = tcfg.args, tcfg.device
        # N > 1: the env-sharded task of the product API -- step() runs the fused step, the observation all-gather beside it and
        # waits for every rank's rows: the observation it returns is the global [world * N, 13] tensor
        tcfg.args = {"shard": "torchrun"} if world > 1 else {"env_id_offset": rank * N, "host_io": host_io}
        tcfg.device = str(dev)
        try:
            t = task_registry.make_task("position_setpoint_task", seed=7, num_envs=N, headless=True)
        finally:
            tcfg.args, tcfg.device = old_args, old_dev
        t.reset()
        t.sim_env.engine.sim_steps.copy_((torch.arange(N, device=dev) % 500).int())
        return t

    h_act = [a.cpu().pin_memory() for a in acts]

    def time_e2e(step_fn):
        for i in range(3):
            step_fn(i)
        barrier()
        t0 = time.perf_counter()
        for i in range(K):
            step_fn(i)
        barrier()
        t = torch.tensor([time.perf_counter() - t0], device=dev, dtype=torch.float64)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return world * N * K / float(t.item())

    # (1) host I/O mode: the one kernel of task.step loads the actions from pinned host memory and
    # stores obs / rewards / terminations / truncations into pinned host memory over PCIe; step()
    # returns when the stream has drained.  Each rank's host consumer gets its own shard.  (N = 1 only: at N > 1 the
    # observation lives in the gather's ring in device memory.)
    e2e_hostio = None
    if world == 1:
        task = make_task(True)
        sink = torch.zeros(4, dtype=torch.float64)

        def e2e_step_hostio(i):
            obs_d, rew_d, term_d, trunc_d, _ = task.step(h_act[i % 8])
            sink[0] += float(rew_d[-1])  # the results are plain CPU tensors: the host reads them in place

        e2e_hostio = time_e2e(e2e_step_hostio)
        task.close()

    # (2) for comparison: device-resident task + explicit pinned-memory copies around step()
    task = make_task(False)
    d_act = torch.empty(N, 4, device=dev)
    h_obs = torch.empty(N, 13).pin_memory()
    h_rew = torch.empty(N).pin_memory()
    h_term = torch.empty(N, dtype=torch.bool).pin_memory()
    h_trunc = torch.empty(N, dtype=torch.bool).pin_memory()

    def e2e_step_memcpy(i):
        d_act.copy_(h_act[i % 8], non_blocking=True)
        obs_d, rew_d, term_d, trunc_d, _ = task.step(d_act)
        h_obs.copy_(obs_d["observations_local"] if world > 1 else obs_d["observations"], non_blocking=True)
        h_rew.copy_(rew_d, non_blocking=True)
        h_term.copy_(term_d, non_blocking=True)
        h_trunc.copy_(trunc_d, non_blocking=True)
        stream.synchronize()  # the user reads the result of every step

    e2e_memcpy = time_e2e(e2e_step_memcpy)
    e2e_gather_ok = None
    if world > 1:  # the global observation the sharded task hands out == the library collective's gather of the ranks' rows
        obs_d = task.step(d_act)[0]
        want = nccl_gather(obs_d["observations_local"].contiguous()).clone()
        okt = torch.tensor([int(torch.equal(obs_d["observations"], want))], device=dev)
        dist.all_reduce(okt, op=dist.ReduceOp.MIN)
        e2e_gather_ok = bool(okt.item())
    task.close()
    e2e_value = e2e_hostio if world == 1 else e2e_memcpy
    h2d = N * 4 * 4
    d2h = N * 13 * 4 + N * 4 + 2 * N

    hp2 = cfg3 = cfg4 = sweep = nav = None
    if not args.no_hp2:
        hp2 = run_hp2_config(dev, world, rank, label="depth+seg camera 64x48, 44-box scene (north_star target config)",
                             metric="depth rays/sec (64x48 depth+seg camera, 44-box scene)", E=args.hp2_envs, K=44, cfg=_CamCfg,
                             frames=max(5, min(K, 50)), extent=5.0, seed=7, cpu_sample_envs=8)
    if not args.no_configs:
        # BASELINE.json configs[2]: navigation_task sensor side -- 270x480 depth camera, 1024-obstacle scene, 8192 envs
        cam3 = type("Cam270x480", (_CamCfg,), {"height": 270, "width": 480})
        cfg3 = run_hp2_config(dev, world, rank, label="BASELINE configs[2]: 270x480 depth+seg camera, 1024 boxes (12,288 triangles) per env",
                              metric="depth rays/sec (270x480 depth+seg camera, 1024-obstacle scene)", E=args.cfg3_envs, K=1024, cfg=cam3,
                              frames=2, extent=8.0, seed=11, cpu_sample_envs=1)
        # BASELINE.json configs[3]: 64x512 LiDAR + segmentation on a fully-actuated octarotor, 16384 envs
        cfg4 = run_hp2_config(dev, world, rank, label="BASELINE configs[3]: 64x512 LiDAR range+seg (OSDome-64), 44 boxes per env",
                              metric="LiDAR rays/sec (64x512 range+seg, 44-box scene)", E=args.cfg4_envs, K=44, cfg=_LidarCfg,
                              frames=5, extent=6.0, seed=13, cpu_sample_envs=2)
        cfg4["dynamics"] = run_hp1_physics(dev, world, rank, robot="base_octarotor", controller=args.cfg4_controller,
                                           N=args.cfg4_envs, substeps=10, steps=20)
        # BASELINE.json configs[4]: env-count sweep of the dynamics + controller step
        sweep = run_hp1_sweep(dev, world, rank, args, [1024, 4096, 16384, 65536, 262144, 1048576])
        nav = run_nav_task(dev, world, rank, args)
    clocks = sampler.stop() if rank == 0 else None

    if rank == 0:
        peaks = {}
        try:
            peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
        except Exception:
            pass
        peak = float(peaks.get("hbm_gbs", 3350.0))
        peak_src = "measured (MEASURED_PEAKS.json hbm_gbs, burst copy)" if "hbm_gbs" in peaks else "fallback 3.35 TB/s (H100 SXM data sheet)"
        # the timed region is K back-to-back launches of the one step kernel bracketed by one CUDA-event pair:
        # average launch duration = region / K.  (A per-launch event pair serialises the launches -- no
        # programmatic-dependent-launch overlap -- and adds the event's own latency: reported separately.)
        main_iso_s = float(main_total.item()) * 1e-3 / Kk
        main_avg_s = total_s / K
        achieved = ALG_BYTES_PER_ENV_STEP * N / main_avg_s / 1e9
        cpu = None
        if world == 1 and not args.no_cpu_baseline:
            v, per, cores, kind, note = time_cpu_reference(ENVS_PER_GPU, 40, 3)
            cpu = {"value": v, "unit": "env-steps/s", "cores": cores, "kind": kind,
                   "sample": f"{ENVS_PER_GPU} envs x 40 steps of the same step, torch CPU fp32: {note}"}
        line = {
            "metric": METRIC, "value": value, "unit": "env-steps/s", "n_gpus": world, "steps": K, "warmup": W,
            "ms_per_step": total_s * 1e3 / K, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "f32", "data": "synthetic",
            "config": workload_config(world, {"envs_per_gpu": N, "global_envs": N * world,
                                              "obs_all_gather": (args.gather if world > 1 else None)}),
            "value_hot_l2": value_hot,
            "value_api_config": value_api,
            "value_obs_gather_sync": value_sync,
            "obs_gather_check": gather_check,
            "obs_gather_multicast": (bool(getattr(gather, "multicast", False)) if gather is not None else None),
            "wall_s_timed_region": t_wall,
            "host_enqueue_us_per_step": 1e6 * t_enqueue / K,
            "roofline": {"bound": "hbm", "kernel": "hp1_step_kernel<4,true,true> (the whole fused step is this one launch)", "achieved": achieved, "peak": peak,
                         "unit": "GB/s", "frac": achieved / peak, "peak_source": peak_src,
                         "algorithmic_bytes_per_launch": ALG_BYTES_PER_ENV_STEP * N,
                         "nvlink_floor_us": ((world - 1) * N * 13 * 4 / 450e9 * 1e6) if world > 1 else None,
                         "kernel_ms_avg": main_avg_s * 1e3,
                         "kernel_ms_isolated_event_pair": main_iso_s * 1e3,
                         "note": "at 65,536 envs the launch is ~14 MB: FP32 dependent-chain latency bound, not HBM bound (DESIGN.md). "
                                 "kernel_ms_avg = timed region / K launches; launches are chained per tile and overlap in flight, so one "
                                 "launch serialised by its own event pair (kernel_ms_isolated_event_pair) takes longer"},
            "cpu_baseline": cpu,
            "e2e": {"value": e2e_value, "unit": "env-steps/s", "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": d2h,
                    "value_memcpy_variant": e2e_memcpy, "sharded_task_obs_equals_nccl": e2e_gather_ok,
                    "api": ("task_registry.make_task('position_setpoint_task', args={'host_io': True}).step(actions): the "
                            "step kernel reads the pinned host actions and writes obs/reward/flags to pinned host memory "
                            "over PCIe (no staging copies), step() returns after the stream drained and the host reads "
                            "its shard in place; value_memcpy_variant = device-resident task + cudaMemcpyAsync both ways.") if world == 1 else
                           ("task_registry.make_task('position_setpoint_task', args={'shard': 'torchrun'}).step(actions) on every rank: pinned "
                            "host actions -> cudaMemcpyAsync -> fused step + observation all-gather (push / wait kernels, awaited every "
                            "step: the global [world*N,13] observation is what step() returns) -> cudaMemcpyAsync of this rank's rows, "
                            "rewards and flags to pinned host memory -> stream synchronise")},
            "gpu_launches": K,
            "clocks": clocks,
            "hp2_depth": hp2,
            "config3_depth_270x480_1024box": cfg3,
            "config4_lidar_64x512_octarotor": cfg4,
            "config5_env_sweep": sweep,
            "navigation_task_e2e": nav,
        }
        print(json.dumps(line))
    if world > 1:
        dist.destroy_process_group()
    return 0


DUMP_MAX_BYTES = 64_000_000  # 64 MB in all, in decimal units (also under 64 MiB)


def dump_outputs(out_dir, e):
    """DIR/<name>.npy (float32; env_index float64) of what the last timed step handed its caller: observation, reward, termination and truncation flags
    and the root state.  Past DUMP_MAX_BYTES in all (.npy headers included) the same fixed, seeded sample of env rows is kept from every
    array, and its row indices are written as env_index.npy.  At N > 1 this is rank 0's shard (its rows of the gathered observation)."""
    import numpy as np

    arrays = {"obs": e.obs, "reward": e.reward, "terminations": e.terminations, "truncations": e.truncations, "root_state": e.root_state}
    arrays = {k: v.detach().cpu().float().numpy() for k, v in arrays.items()}
    n = len(arrays["reward"])
    row_bytes = sum(a[0].nbytes if a.ndim > 1 else a.itemsize for a in arrays.values())
    budget = DUMP_MAX_BYTES - (64 << 10)  # room for the six .npy headers
    if n * row_bytes > budget:
        rows = np.sort(np.random.default_rng(0).choice(n, budget // (row_bytes + 8), replace=False))  # + 8: env_index is float64
        arrays = {k: a[rows] for k, a in arrays.items()}
        arrays["env_index"] = rows.astype(np.float64)
    os.makedirs(out_dir, exist_ok=True)
    for k, a in arrays.items():
        np.save(os.path.join(out_dir, f"{k}.npy"), np.ascontiguousarray(a))


class _CamCfg:
    """BaseDepthCameraConfig (config/sensor_config/camera_config/base_depth_camera_config.py:16-52): depth + segmentation, normalised"""
    sensor_type, num_sensors, height, width = "camera", 1, 48, 64
    horizontal_fov_deg, max_range, min_range = 87.0, 10.0, 0.2
    calculate_depth, return_pointcloud, pointcloud_in_world_frame = True, False, False
    segmentation_camera, normalize_range = True, True
    far_out_of_range_value, near_out_of_range_value = 10.0, -10.0
    euler_frame_rot_deg = [-90.0, 0, -90.0]


class _LidarCfg:
    """OSDome_64_Config (config/sensor_config/lidar_config/osdome_64_config.py:4-32): 64 x 512, az +-180, el 0..90, range + segmentation"""
    sensor_type, num_sensors, height, width = "lidar", 1, 64, 512
    horizontal_fov_deg_min, horizontal_fov_deg_max, vertical_fov_deg_min, vertical_fov_deg_max = -180, 180, 0, 90
    max_range, min_range = 20.0, 0.5
    return_pointcloud, pointcloud_in_world_frame, segmentation_camera, normalize_range = False, False, True, True
    far_out_of_range_value, near_out_of_range_value = 20.0, -20.0
    euler_frame_rot_deg = [0.0, 0.0, 0.0]


def _peak_hbm():
    try:
        peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
        return float(peaks["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs, burst copy)"
    except Exception:
        return 3350.0, "fallback 3.35 TB/s (H100 SXM data sheet)"


def cpu_ray_baseline(sensor, scene_np, robot_np, sample_envs):
    """rays/s of the oracle's brute-force closest hit (oracle/hp2_oracle.c, one thread) on `sample_envs` envs of the same scene
    and sensor -- a `port`: the reference's own ray query is Warp's BVH (warp-lang 1.0.0, not installable here)"""
    import numpy as np

    from oracle import hp2_oracle as RO

    E = sample_envs
    offs = np.arange(0, 12 * (len(scene_np["templates"]) + 1), 12, dtype=np.int32)
    nt = 12 * len(scene_np["templates"])
    tris, segs, cnt = RO.build_world_tris(scene_np["pose"][:E, :, :7], scene_np["tm"][:E], scene_np["ctr"][:E], offs,
                                          np.concatenate(scene_np["templates"]), np.zeros(nt, np.int32), np.ones(nt, np.int32),
                                          scene_np["tm"].shape[1] * 12)
    so = RO.Hp2oSensor()
    for f, _ in RO.Hp2oSensor._fields_:
        if hasattr(sensor.c, f):
            setattr(so, f, getattr(sensor.c, f))
    mount = np.zeros((E, 1, 7), np.float32)
    mount[..., 6] = 1
    table = sensor.ray_table.cpu().numpy() if getattr(sensor, "ray_table", None) is not None else None
    t0 = time.perf_counter()
    RO.cast(so, robot_np[:E, :7], mount, table, tris, segs, cnt)
    dt = time.perf_counter() - t0
    rays = E * sensor.c.height * sensor.c.width
    return {"value": rays / dt, "unit": "rays/s", "cores": 1, "kind": "port",
            "sample": f"{E} env(s) x {sensor.c.height}x{sensor.c.width} rays against {int(cnt[0])} triangles, brute-force closest hit "
                      f"(oracle/hp2_oracle.c, 1 thread, {dt:.2f} s); the reference's Warp BVH query is not installable"}


def run_hp2_config(dev, world, rank, *, label, metric, E, K, cfg, frames, extent, seed, cpu_sample_envs=0):
    """rays/sec of the ray-caster on one BASELINE.json sensor config: E envs per GPU, K randomly posed boxes per env (12 triangles
    each), one sensor per env.  Synthetic scenes; the E scenes together exceed L2, so no flush is needed between frames."""
    import numpy as np
    import torch
    import torch.distributed as dist

    from aerial_gym_simulator_b200.hp2 import RayScene, RaySensor, box_obb, box_triangles

    H, W = cfg.height, cfg.width
    g = torch.Generator().manual_seed(seed + rank)
    sizes = torch.rand(5, 3, generator=g) * 1.2 + 0.15
    templates = [box_triangles(s_.tolist()) for s_ in sizes]
    pose = torch.zeros(E, K, 13)
    pose[..., 0:3] = (torch.rand(E, K, 3, generator=g) * 2 - 1) * extent
    q = torch.randn(E, K, 4, generator=g)
    pose[..., 3:7] = q / q.norm(dim=-1, keepdim=True)
    tm = torch.randint(0, 5, (E, K), generator=g).numpy()
    ctr = (100 + torch.arange(E * K).reshape(E, K) % 100000).numpy()
    scene = RayScene(templates, [0] * 5, [1] * 5, tm, ctr, pose.to(dev), dev,
                     tmpl_obb=np.stack([box_obb(s_.tolist()) for s_ in sizes]))
    robot = torch.zeros(E, 13)
    robot[:, 0:3] = (torch.rand(E, 3, generator=g) * 2 - 1) * (extent * 0.8)
    rq = torch.randn(E, 4, generator=g)
    robot[:, 3:7] = rq / rq.norm(dim=-1, keepdim=True)
    robot_d = robot.to(dev)
    pix = torch.zeros(E, 1, H, W, device=dev)
    seg = torch.zeros(E, 1, H, W, dtype=torch.int32, device=dev)
    sensor = RaySensor(cfg, scene, robot_d, pix, seg)
    stream = torch.cuda.current_stream(dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    scene.update()
    e1.record(stream)
    torch.cuda.synchronize(dev)
    build_ms = e0.elapsed_time(e1)
    for _ in range(3 if frames > 3 else 1):
        sensor.capture()
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize(dev)
    e0.record(stream)
    for _ in range(frames):
        sensor.capture()
    e1.record(stream)
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize(dev)
    t = torch.tensor([e0.elapsed_time(e1)], device=dev, dtype=torch.float64)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    sec = float(t.item()) * 1e-3
    rays = E * H * W
    hit_frac = float((seg >= 0).float().mean())
    out_bytes = rays * 8
    scene_bytes = E * (K * 12 * 48 + (2 * scene.P - 1) * 32 + max(scene.P, 4) * 4)
    peak, peak_src = _peak_hbm()
    achieved = (out_bytes + scene_bytes) * frames / sec / 1e9
    cpu = None
    if cpu_sample_envs and rank == 0 and world == 1:
        cpu = cpu_ray_baseline(sensor, {"templates": templates, "pose": pose.numpy(), "tm": tm, "ctr": ctr}, robot.numpy(), cpu_sample_envs)
    res = {
        "metric": metric, "value": world * rays * frames / sec, "unit": "rays/s", "workload": label, "envs_per_gpu": E, "image": [H, W],
        "objects_per_env": K, "triangles_per_env": K * 12, "frames": frames, "ms_per_frame": sec * 1e3 / frames, "hit_fraction": hit_frac,
        "scene_update_ms_all_envs": build_ms, "gpu_launches": frames, "n_gpus": world, "scaling": "weak",
        "traversal": ("tile path, scene staged into shared memory by TMA bulk copies" if scene.P <= 128 else
                      ("tile path, object records in shared memory + candidate slabs from L2 (scene larger than shared memory)" if cfg.sensor_type != "lidar"
                       else "per-ray BVH traversal" + (" from shared memory" if scene.P * 12 * 48 < 200000 else " from L2"))),
        "roofline": {"bound": "hbm (nominal: FP32 traversal / intersection issue binds, see DESIGN 6)", "achieved": achieved, "peak": peak, "unit": "GB/s",
                     "frac": achieved / peak, "peak_source": peak_src, "algorithmic_bytes_per_frame": out_bytes + scene_bytes,
                     "note": "8 B/ray written (depth or range + segmentation) + every env's scene (48-byte triangle slabs + BVH) read once per frame"},
        "cpu_baseline": cpu,
    }
    del sensor, scene, pix, seg
    torch.cuda.empty_cache()
    return res


def run_hp1_physics(dev, world, rank, *, robot, controller, N, substeps, steps):
    """env-steps/sec of the HP1 physics launch alone (agx_hp1_physics_step, `substeps` fused physics steps per env step) for a robot /
    controller pair from the registry -- the dynamics side of BASELINE config #4 (fully-actuated octarotor, 16,384 envs)"""
    import torch
    import torch.distributed as dist

    import aerial_gym_simulator_b200.robots  # noqa: F401
    from aerial_gym_simulator_b200.config.env_config import EmptyEnvCfg
    from aerial_gym_simulator_b200.config.sim_config import BaseSimConfig
    from aerial_gym_simulator_b200.hp1 import Hp1Engine
    from aerial_gym_simulator_b200.registry._core import robot_registry

    rb, _ = robot_registry.make_robot(robot, controller, EmptyEnvCfg, "cpu")
    spec = rb.make_spec(BaseSimConfig, EmptyEnvCfg)
    eng = Hp1Engine(spec, N, dev, seed=5, env_id_offset=rank * N, materialize_derived=True)
    eng.reset(torch.ones(N, dtype=torch.bool, device=dev))
    eng.refresh()
    g = torch.Generator(device=dev).manual_seed(9 + rank)
    acts = (torch.rand(N, spec.num_actions, generator=g, device=dev) * 2 - 1).contiguous()
    if spec.num_actions == 7:  # pose command: position + unit quaternion
        acts[:, 3:7] = torch.nn.functional.normalize(acts[:, 3:7], dim=1)
    stream = torch.cuda.current_stream(dev)
    for _ in range(5):
        eng.physics_step(acts, physics_steps=substeps)
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize(dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(steps):
        eng.physics_step(acts, physics_steps=substeps)
    e1.record(stream)
    torch.cuda.synchronize(dev)
    t = torch.tensor([e0.elapsed_time(e1)], device=dev, dtype=torch.float64)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    sec = float(t.item()) * 1e-3
    assert torch.isfinite(eng.root_state).all()
    return {"metric": f"env-steps/sec ({robot} + {controller}, {substeps} physics sub-steps per env step, physics launch only)",
            "value": world * N * steps / sec, "unit": "env-steps/s", "envs_per_gpu": N, "ms_per_env_step": sec * 1e3 / steps,
            "physics_substeps_per_s": world * N * steps * substeps / sec, "gpu_launches": steps, "num_motors": spec.num_motors}


def run_hp1_sweep(dev, world, rank, args, sizes):
    """BASELINE config #5: env-count sweep of the fused position-task step (dynamics + controller + task epilogue), N > 1 with the
    observation all-gather.  Per size: one replica set sized to exceed L2 (or 2 replicas at the large sizes), K steps."""
    import torch
    import torch.distributed as dist

    from aerial_gym_simulator_b200.distributed import ObsAllGather, PipelinedObsGather
    from aerial_gym_simulator_b200.hp1 import Hp1Engine, MultirotorSpec

    peak, _ = _peak_hbm()
    out = []
    for N in sizes:
        R = max(2, min(16, (160 << 20) // (N * 190)))  # ~190 B of state / outputs per env: replicas until the set exceeds L2
        K = max(20, min(args.steps, 200))
        engines = []
        for rep in range(R):
            e = Hp1Engine(MultirotorSpec(), N, dev, seed=1 + rep, env_id_offset=rank * N, materialize_derived=False)
            e.reset(torch.ones(N, dtype=torch.bool, device=dev))
            e.refresh()
            e.sim_steps.copy_((torch.arange(N, device=dev) % 500).int())
            engines.append(e)
        chained = bool(engines[0].lib.agx_hp1_task_step_is_chained(engines[0]._cfg_ref, engines[0]._buf_ref))
        g = torch.Generator(device=dev).manual_seed(77 + rank)
        acts = [(torch.rand(N, 4, generator=g, device=dev) * 2 - 1).contiguous() for _ in range(4)]
        gather, nccl = None, None
        if world > 1:
            if args.gather != "nccl" and (N * 52) % 16 == 0:
                gather = PipelinedObsGather(N, 13, dev, num_buffers=4, max_ctas=args.gather_ctas)
                for e in engines:
                    e.attach_obs_gather(gather)
            else:
                nccl = ObsAllGather(N, 13, world * N, dev)
        stream = torch.cuda.current_stream(dev)

        def loop(n):
            for i in range(n):
                e = engines[i % R]
                e.position_task_step(acts[i % 4])
                if nccl is not None:
                    nccl(e.obs)
            if gather is not None:
                gather.fence()
                gather.wait()

        loop(max(R, 5))
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize(dev)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        loop(K)
        e1.record(stream)
        torch.cuda.synchronize(dev)
        t = torch.tensor([e0.elapsed_time(e1)], device=dev, dtype=torch.float64)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        sec = float(t.item()) * 1e-3
        if gather is not None:
            gather.check()
        engines[0].check()
        val = world * N * K / sec
        out.append({"envs_per_gpu": N, "global_envs": N * world, "value": val, "unit": "env-steps/s", "us_per_step": sec * 1e6 / K, "steps": K,
                    "replicas": R, "path": "single launch, chained per tile" if chained else "two launches (grid larger than one resident wave)",
                    "roofline_frac": ALG_BYTES_PER_ENV_STEP * N * K / sec / 1e9 / peak,
                    "nvlink_floor_us": ((world - 1) * N * 52 / 450e9 * 1e6) if world > 1 else None})
        for e in engines:
            if gather is not None:
                e.attach_obs_gather(None)
        del engines, gather, nccl
        torch.cuda.synchronize(dev)
        torch.cuda.empty_cache()
    return out


def run_nav_task(dev, world, rank, args):
    """navigation_task end to end through the task API at its shipped configuration (config/task_config/navigation_task_config.py:
    lmf2 + lmf2_velocity_control, env_with_obstacles = 44 boxes, 135x240 depth camera, VAE latents, 10 physics sub-steps per env
    step) -- env-steps/s of task.step(actions) with device-resident actions."""
    import torch
    import torch.distributed as dist

    import aerial_gym_simulator_b200.task  # noqa: F401
    from aerial_gym_simulator_b200.registry.task_registry import task_registry

    N = args.nav_envs
    tcfg = task_registry.get_task_config("navigation_task")
    old = (tcfg.args, tcfg.device) if hasattr(tcfg, "args") else (None, tcfg.device)
    try:
        tcfg.device = str(dev)
        t0 = time.perf_counter()
        task = task_registry.make_task("navigation_task", seed=3 + rank, num_envs=N, headless=True)
        build_s = time.perf_counter() - t0
    finally:
        tcfg.device = old[1]
    task.reset()
    A = task.task_config.action_space_dim
    g = torch.Generator(device=dev).manual_seed(5 + rank)
    acts = [(torch.rand(N, A, generator=g, device=dev) * 2 - 1) for _ in range(4)]
    K = max(10, min(args.steps, 50))
    for i in range(5):
        task.step(acts[i % 4])
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize(dev)
    t0 = time.perf_counter()
    for i in range(K):
        task.step(acts[i % 4])
    torch.cuda.synchronize(dev)
    t = torch.tensor([time.perf_counter() - t0], device=dev, dtype=torch.float64)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    sec = float(t.item())
    env = task.sim_env
    rays = N * env.sensor.c.height * env.sensor.c.width if getattr(env, "sensor", None) is not None else 0
    # where the env step goes: the three device-side stages alone (CUDA events), the rest is the task's torch / host code
    def stage_ms(fn, reps=10):
        fn()
        torch.cuda.synchronize(dev)
        a0, a1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a0.record()
        for _ in range(reps):
            fn()
        a1.record()
        torch.cuda.synchronize(dev)
        return a0.elapsed_time(a1) / reps
    act_t = task.action_transformation_function(acts[0])
    breakdown = {"physics_x10_plus_collision_ms": stage_ms(lambda: env.step(actions=act_t)), "render_depth_ms": stage_ms(lambda: env.render()),
                 "vae_encode_ms": stage_ms(task.process_image_observation)}
    res = {"metric": "env-steps/sec (navigation_task: lmf2, env_with_obstacles, 135x240 depth camera + VAE, 10 physics sub-steps)",
           "value": world * N * K / sec, "unit": "env-steps/s", "envs_per_gpu": N, "ms_per_env_step": sec * 1e3 / K, "steps": K,
           "rays_per_s_inside": world * rays * K / sec, "construction_s": build_s,
           "step_mode": getattr(env, "step_mode", "launch per kernel"), "breakdown": breakdown,
           "timing": "host wall clock around K x task.step, synchronised"}
    task.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--envs", type=int, default=ENVS_PER_GPU, help="envs per GPU (default: BASELINE configs[1])")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR",
                    help="write the observation, reward, flags and root state of the last timed step as DIR/<name>.npy (float32, at most "
                         "64 MB: a fixed, seeded sample of env rows beyond that; at N > 1 rank 0's shard); inputs are seeded, so runs with the "
                         "same arguments compare output for output")
    ap.add_argument("--gather", default="pipelined", choices=["pipelined", "sync", "nccl"],
                    help="N>1 observation all-gather: hand-written NVLink push / wait kernels beside the chained steps, the push of "
                         "step t overlapping step t+1 (default; actions are pre-generated, as at N=1); the same kernels awaited "
                         "after every step; or NCCL's all_gather_into_tensor after every step")
    ap.add_argument("--gather-ctas", type=int, default=24, help="CTAs of the push kernel (it shares the GPU with the step kernel)")
    ap.add_argument("--no-hp2", action="store_true", help="skip the secondary depth rays/sec measurement")
    ap.add_argument("--hp2-envs", type=int, default=8192)
    ap.add_argument("--no-configs", action="store_true", help="skip the BASELINE configs[2..4] sub-lines and the navigation_task line")
    ap.add_argument("--cfg3-envs", type=int, default=8192)
    ap.add_argument("--cfg4-envs", type=int, default=16384)
    ap.add_argument("--cfg4-controller", default="rov_fully_actuated_control", help="7-D pose command, FullyActuatedController")
    ap.add_argument("--nav-envs", type=int, default=1024)
    ap.add_argument("--multi-gpu-sublines", action="store_true",
                    help="N > 1: also run the single-GPU sub-lines (hp2_depth, configs[2..4], navigation_task) on every rank; by default they are "
                         "measured at N = 1 only -- the N > 1 line is the headline workload with its all-gather and the sharded-task e2e")
    args = ap.parse_args()
    if int(os.environ.get("WORLD_SIZE", "1")) > 1 and not args.multi_gpu_sublines:
        args.no_hp2 = args.no_configs = True
    # stdout carries exactly ONE JSON line: everything else a library prints there (NCCL's version banner, the reference's logger)
    # goes to stderr -- file descriptor 1 is pointed at stderr for the run and the line is written to the real stdout at the end
    sys.stdout.flush()
    real_stdout = os.dup(1)
    os.dup2(2, 1)
    lines = []
    orig_print = print

    def capture_print(*a, **k):
        if k.get("file") in (None, sys.stdout):
            lines.append(" ".join(str(x) for x in a))
        else:
            orig_print(*a, **k)

    import builtins
    builtins.print = capture_print
    try:
        rc = run_reference_arm(args) if args.impl == "reference" else run_ours(args)
    finally:
        builtins.print = orig_print
        sys.stdout.flush()
        os.dup2(real_stdout, 1)
        os.close(real_stdout)
    for ln in lines:
        if ln.startswith("{"):
            print(ln, flush=True)
        else:
            sys.stderr.write(ln + "\n")
    return rc


if __name__ == "__main__":
    sys.exit(main())
