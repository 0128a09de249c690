"""In-tree build of libaerial_gym_b200.so (nvcc, sm_90a only: H100).

``python -m aerial_gym_simulator_b200._build`` or ``__graft_entry__.build()``.
The .so and the objects under build/ are git-ignored build products."""
import os
import subprocess
import sys
import sysconfig

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, "csrc")
LIB = os.path.join(PKG, "libaerial_gym_b200.so")
# hp2_raycast.cu is compiled with -fmad=false: its ray/triangle arithmetic is written with explicit
# fmaf() so that the C oracle (oracle/hp2_oracle.c, -ffp-contract=off) is bit-reproducible.
UNITS = [
    ("agx_common.cu", []),
    # hp1: 2-ulp division / sqrt (no slow-path branches): the step is a long dependent chain per warp, every instruction counts
    ("hp1.cu", ["-prec-div=false", "-prec-sqrt=false"]),  # AGX_FAST_TRIG: 3x parity error -> off
    ("hp1_aux.cu", []),
    ("articulated.cu", []),
    ("articulated_prismatic.cu", []),
    ("lidar_nav.cu", []),
    # device-RNG units: no FMA contraction, so "lo + (hi - lo) u" and the noise model round like their numpy oracles
    ("sensor_noise.cu", ["-fmad=false"]),
    ("obstacles.cu", ["-fmad=false"]),
    ("e2e_task.cu", []),
    ("sim2real.cu", []),
    ("disturbance.cu", ["-fmad=false"]),
    ("hp2_raycast.cu", ["-fmad=false"]),
    ("p2p_allgather.cu", []),
]
# the CPython extension Hp1Engine calls the per-step entry through (csrc/hostcall.cpp): host code only, no device code
HOSTCALL_SRC = os.path.join(CSRC, "hostcall.cpp")
HOSTCALL = os.path.join(PKG, "_hostcall" + (sysconfig.get_config_var("EXT_SUFFIX") or ".so"))
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
]


def _nvcc():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    raise RuntimeError("nvcc not found")


def cuda_tool(name):
    """a CUDA toolkit binary (cuobjdump, ...) from the same toolkit as nvcc"""
    nvcc = _nvcc()
    return os.path.join(os.path.dirname(nvcc), name) if os.path.isabs(nvcc) else name


def sources():
    return [os.path.join(CSRC, u) for u, _ in UNITS if os.path.exists(os.path.join(CSRC, u))]


def needs_build():
    if not os.path.exists(LIB) or not os.path.exists(HOSTCALL):
        return True
    t = min(os.path.getmtime(LIB), os.path.getmtime(HOSTCALL))
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(PKG, "..", "include", "aerial_gym_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    nvcc = _nvcc()
    objs = []
    os.makedirs(os.path.join(PKG, "build"), exist_ok=True)
    for unit, extra in UNITS:
        src = os.path.join(CSRC, unit)
        if not os.path.exists(src):
            continue
        obj = os.path.join(PKG, "build", unit.replace(".cu", ".o"))
        cmd = [nvcc] + NVCC_FLAGS + extra + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if verbose or r.returncode:
            sys.stderr.write(r.stdout + r.stderr)
        if r.returncode:
            raise RuntimeError(f"nvcc failed for {unit}")
        objs.append(obj)
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-o", LIB] + objs
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("link failed")
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-shared",
           "-I", sysconfig.get_paths()["include"], HOSTCALL_SRC, "-o", HOSTCALL]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("nvcc failed for hostcall.cpp")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
