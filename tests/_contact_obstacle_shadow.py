"""Build + load the CPU shadow of the obstacle-obstacle contact (tests/csrc/contact_obstacle_shadow.cu).  Test infrastructure only."""
import ctypes as C
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "csrc", "contact_obstacle_shadow.cu")
LIB = os.path.join(HERE, "_build", "libagx_contact_obstacle_shadow.so")
_CSRC = os.path.join(HERE, "..", "aerial_gym_simulator_b200", "csrc")
_DEPS = [SRC, os.path.join(_CSRC, "contact_core.cuh"), os.path.join(_CSRC, "agx_math.cuh"),
         os.path.join(HERE, "..", "include", "aerial_gym_b200.h")]
_lib = None


def build(force=False):
    if not force and os.path.exists(LIB) and all(os.path.getmtime(d) <= os.path.getmtime(LIB) for d in _DEPS):
        return LIB
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    # host code only; no FMA contraction, as in the device unit (-fmad=false)
    cmd = [nvcc, "-x", "cu", "-DAGX_HOST_SHADOW", "-O2", "-std=c++17", "--expt-relaxed-constexpr", "-Wno-deprecated-gpu-targets",
           "-Xcompiler", "-fPIC,-ffp-contract=off", "-shared", "-o", LIB, SRC]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode:
        raise RuntimeError("obstacle contact shadow build failed:\n" + r.stdout + r.stderr)
    return LIB


def load():
    global _lib
    if _lib is None:
        from aerial_gym_simulator_b200 import _lib as A
        lib = C.CDLL(build())
        lib.shadow_obstacle_obstacle.restype = None
        lib.shadow_obstacle_obstacle.argtypes = [C.c_int, C.c_int, C.POINTER(A.AgxContactParams), C.c_void_p, C.c_int, C.c_void_p,
                                                 C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib = lib
    return _lib
