"""Where the time of one chained position-task step goes (bench.py's flagship loop: 65,536 envs, 16 rotating replicas, lean engines).

    python tools/build_variant.py timeline --hp1 "-DAGX_TIMELINE"
    python tools/step_breakdown.py --timeline-lib tools/dbg/libagx_timeline.so [--root DIR] [--envs 65536]

Prints one JSON line:
- handshake (the AGX_TIMELINE build's per-warp %globaltimer stamps; the last step of a run of chained steps, so it overlaps its
  predecessor as in the timed loop): median per warp of each phase -- step index known (claim), both waits done, first state loads
  arrived, rest of the step -- for cold16 (16 replicas in turn) and hot (one replica back to back);
- host enqueue per step: the Python body of position_task_step with the library call replaced by a no-op, the library call (the
  _hostcall extension; ctypes in a tree without it) with the same arguments to a C function that returns at once, the C entry up to
  its launch and cudaLaunchKernelEx of an empty kernel with the chained step's launch configuration and its parameter block and with
  AgxHp1Buffers alone (agx_dbg_host_costs, same build), and the whole call (position_task_step of the product library, as
  bench.py's host_enqueue_us_per_step).
--root: the checkout whose package is imported (an A/B against another tree's build); the timeline-lib phase runs in a subprocess."""
import argparse
import ctypes as C
import functools
import json
import os
import statistics
import subprocess
import sys
import time

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R = 16


def _engines(root, N):
    sys.path.insert(0, root)
    import torch

    from aerial_gym_simulator_b200.hp1 import Hp1Engine, MultirotorSpec
    dev = torch.device("cuda:0")
    engines = []
    for rep in range(R):
        e = Hp1Engine(MultirotorSpec(), N, dev, seed=1 + rep, materialize_derived=False)
        e.reset(torch.ones(N, dtype=torch.bool, device=dev))
        e.refresh()
        e.sim_steps.copy_((torch.arange(N, device=dev) % 500).int())
        engines.append(e)
    g = torch.Generator(device=dev).manual_seed(1234)
    acts = [(torch.rand(N, 4, generator=g, device=dev) * 2 - 1).contiguous() for _ in range(8)]
    return torch, engines, acts


def _loop(engines, acts, k, rotate, i0=0):
    for i in range(i0, i0 + k):
        engines[i % R if rotate else 0].position_task_step(acts[i % 8])


def timeline_phase(root, N, reps):
    """runs with AGX_LIB_PATH = an AGX_TIMELINE build"""
    import numpy as np
    torch, engines, acts = _engines(root, N)
    from aerial_gym_simulator_b200 import _lib
    lib = _lib.load()
    lib.agx_dbg_timeline.argtypes = [C.c_void_p]
    W = (N + 31) // 32
    out = {}
    for mode, rotate in (("cold16", True), ("hot", False)):
        _loop(engines, acts, 64, rotate)
        torch.cuda.synchronize()
        ph = {k: [] for k in ("claim", "waits", "first_loads", "rest", "warp_lifetime")}
        for rep in range(reps):
            _loop(engines, acts, 2 * R, rotate, i0=rep)  # the last launch runs overlapped with its predecessor, as in the timed loop
            torch.cuda.synchronize()
            t = np.zeros((7, 8192), dtype=np.uint64)
            _lib.check(lib.agx_dbg_timeline(t.ctypes.data_as(C.c_void_p)), "agx_dbg_timeline")
            t = t[:, :W].astype(np.int64)
            ph["claim"].append(np.median(t[4] - t[0]))
            ph["waits"].append(np.median(t[5] - t[4]))
            ph["first_loads"].append(np.median(t[6] - t[5]))
            ph["rest"].append(np.median(t[3] - t[6]))
            ph["warp_lifetime"].append(np.median(t[3] - t[0]))
        out[mode] = {k: round(float(np.median(v)) / 1e3, 3) for k, v in ph.items()}
        out[mode]["unit"] = "us, median per warp (median over %d steps)" % reps
    for e in engines:
        e.check()
    host = None
    if hasattr(lib, "agx_dbg_host_costs"):
        lib.agx_dbg_host_costs.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_double)]
        e = engines[0]
        res = (C.c_double * 3)()
        best = [1e9] * 3
        for _ in range(5):
            _lib.check(lib.agx_dbg_host_costs(C.addressof(e.cfg), C.addressof(e._buf), e._stream(), 2000, res), "agx_dbg_host_costs")
            best = [min(b, r) for b, r in zip(best, res)]
        host = {"c_entry_before_launch_us": round(best[0], 3), "launch_empty_kernel_1252B_params_us": round(best[1], 3),
                "launch_empty_kernel_264B_params_us": round(best[2], 3),
                "param_bytes": C.sizeof(e.cfg) + C.sizeof(e._buf) + 8}
    return {"handshake": out, "host_c": host}


def host_phase(root, N, steps):
    torch, engines, acts = _engines(root, N)
    from aerial_gym_simulator_b200 import _lib
    lib = _lib.load()
    stream = torch.cuda.current_stream()
    _loop(engines, acts, 64, True)
    torch.cuda.synchronize()
    # (a) the whole call, as bench.py times it: K rotating steps enqueued, then the device drained
    whole, dev_us = [], []
    for rep in range(7):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        e0.record(stream)
        _loop(engines, acts, steps, True)
        e1.record(stream)
        t1 = time.perf_counter()
        torch.cuda.synchronize()
        whole.append((t1 - t0) * 1e6 / steps)
        dev_us.append(e0.elapsed_time(e1) * 1e3 / steps)
    for e in engines:
        e.check()
    # (b) the Python body: the library call replaced by a no-op Python function (its own call cost is reported beside it)
    name = "_task_step_at" if hasattr(engines[0], "_task_step_at") else "_task_step"
    real = [getattr(e, name) for e in engines]
    chain = [e._chain_T for e in engines]

    def noop(*a):
        return 0

    for e in engines:
        setattr(e, name, noop)
    n = 20000
    body = []
    for _ in range(5):
        t0 = time.perf_counter()
        _loop(engines, acts, n, True)
        body.append((time.perf_counter() - t0) * 1e6 / n)
    t0 = time.perf_counter()
    for _ in range(n):
        noop(1, 2, 3, 4)
    noop_us = (time.perf_counter() - t0) * 1e6 / n
    for e, f, T in zip(engines, real, chain):
        setattr(e, name, f)
        e._chain_T = T  # the no-op calls launched nothing
    # (c) the same call with the same argument values to a C function that returns at once (agx_abi_version: the extra register
    # arguments are ignored): the _hostcall extension, or a ctypes call (a tree without it)
    e = engines[0]
    f, nop = getattr(e, name), C.cast(lib.agx_abi_version, C.c_void_p).value
    proto = functools.partial(f.func, nop) if isinstance(f, functools.partial) else C.CFUNCTYPE(C.c_int, *f.argtypes)(nop)
    args = (e._cfg_addr, e._buf_addr, e._stream(), 0) if hasattr(e, "_cfg_addr") else (e._cfg_ref, e._buf_ref, e._stream())
    ct = []
    for _ in range(5):
        t0 = time.perf_counter()
        for _ in range(n):
            proto(*args)
        ct.append((time.perf_counter() - t0) * 1e6 / n)
    return {"whole_call_us": round(statistics.median(whole), 3), "whole_call_us_runs": [round(x, 3) for x in whole],
            "device_us_per_step": round(statistics.median(dev_us), 3),
            "python_body_us": round(min(body), 3), "python_noop_call_us": round(noop_us, 3), "call_us": round(min(ct), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=65536)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--root", default=HERE)
    ap.add_argument("--timeline-lib")
    ap.add_argument("--phase", choices=("all", "timeline"), default="all")
    a = ap.parse_args()
    root = os.path.abspath(a.root)
    if a.phase == "timeline":
        print(json.dumps(timeline_phase(root, a.envs, a.reps)), flush=True)
        return
    out = {"root": os.path.basename(root), "envs": a.envs}
    if a.timeline_lib:
        env = dict(os.environ, AGX_LIB_PATH=os.path.abspath(a.timeline_lib))
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--phase", "timeline", "--root", root, "--envs", str(a.envs),
                            "--reps", str(a.reps)], env=env, capture_output=True, text=True)
        if r.returncode:
            sys.stderr.write(r.stdout[-2000:] + r.stderr[-4000:])
            raise SystemExit("timeline phase failed")
        out.update(json.loads(r.stdout.strip().splitlines()[-1]))
    out["host"] = host_phase(root, a.envs, a.steps)
    import torch
    p = torch.cuda.get_device_properties(0)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    out["gpu"] = q.stdout.strip() or p.name
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
