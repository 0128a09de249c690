"""Build + load the CPU shadow of the articulated step with the joint forces (tests/csrc/articulated_joint_force_shadow.cu).  Test
infrastructure only."""
import ctypes as C
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "csrc", "articulated_joint_force_shadow.cu")
LIB = os.path.join(HERE, "_build", "libagx_articulated_joint_force_shadow.so")
_CSRC = os.path.join(HERE, "..", "aerial_gym_simulator_b200", "csrc")
_DEPS = [SRC] + [os.path.join(_CSRC, f) for f in ("articulated_core.cuh", "hp1_core.cuh", "disturbance_core.cuh", "agx_math.cuh")] + \
        [os.path.join(HERE, "..", "include", "aerial_gym_b200.h")]
_lib = None


def build(force=False):
    if not force and os.path.exists(LIB) and all(os.path.getmtime(d) <= os.path.getmtime(LIB) for d in _DEPS):
        return LIB
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    tmp = f"{LIB}.{os.getpid()}.tmp"
    cmd = [nvcc, "-x", "cu", "-DAGX_HOST_SHADOW", "-O2", "-std=c++17", "--expt-relaxed-constexpr", "-Wno-deprecated-gpu-targets",
           "-Xcompiler", "-fPIC,-ffp-contract=off", "-shared", "-o", tmp, SRC]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode:
        raise RuntimeError("articulated joint force shadow build failed:\n" + r.stdout + r.stderr)
    os.replace(tmp, LIB)
    return LIB


def load():
    global _lib
    if _lib is None:
        from aerial_gym_simulator_b200 import _lib as A
        lib = C.CDLL(build())
        lib.shadow_art_step_joint_force.restype = C.c_int
        lib.shadow_art_step_joint_force.argtypes = [C.POINTER(A.AgxHp1Config), C.POINTER(A.AgxHp1Buffers), C.POINTER(A.AgxArticulation),
                                                    C.POINTER(A.AgxJointEffort), C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib = lib
    return _lib
