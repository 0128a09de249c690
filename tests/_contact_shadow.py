"""Build + load the CPU shadow of the contact solves (tests/csrc/contact_shadow.cu).  Test infrastructure only."""
import ctypes as C
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "csrc", "contact_shadow.cu")
LIB = os.path.join(HERE, "_build", "libagx_contact_shadow.so")
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
        raise RuntimeError("contact shadow build failed:\n" + r.stdout + r.stderr)
    return LIB


def load():
    global _lib
    if _lib is None:
        from aerial_gym_simulator_b200 import _lib as A
        lib = C.CDLL(build())
        P, i, ll, v = C.POINTER(A.AgxContactParams), C.c_int, C.c_longlong, C.c_void_p
        argtypes = {
            "shadow_contact_solve": [i, P, v, i, v, v, v, v],
            "shadow_contact_select": [i, v, v, v],
            "shadow_contact_solve_moving": [i, P, v, i, v, v, v, v, v],
            "shadow_obstacle_point_vel": [v, v, v],
            "shadow_contact_solve_dynamic": [i, P, v, i, v, v, v, i, v, i, i, v, v, v, v],
            "shadow_obstacle_ground": [ll, P, v, i, v, v, v, v, v, v, v],
            "shadow_obstacle_obstacle": [i, i, P, v, i, v, v, v, v, v],
        }
        for name, args in argtypes.items():
            f = getattr(lib, name)
            f.argtypes = args
            f.restype = C.c_int if name == "shadow_contact_select" else None
        _lib = lib
    return _lib
