"""Build + load the CPU shadow of the articulated-multirotor kernels (tests/csrc/articulated_shadow.cu).  Test infrastructure only."""
import ctypes as C
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "csrc", "articulated_shadow.cu")
LIB = os.path.join(HERE, "_build", "libagx_articulated_shadow.so")
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
    # host code only; no FMA contraction, as in the other shadows
    cmd = [nvcc, "-x", "cu", "-DAGX_HOST_SHADOW", "-O2", "-std=c++17", "--expt-relaxed-constexpr", "-Wno-deprecated-gpu-targets",
           "-Xcompiler", "-fPIC,-ffp-contract=off", "-shared", "-o", tmp, SRC]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode:
        raise RuntimeError("articulated shadow build failed:\n" + r.stdout + r.stderr)
    os.replace(tmp, LIB)
    return LIB


def load():
    global _lib
    if _lib is None:
        from aerial_gym_simulator_b200 import _lib as A
        lib = C.CDLL(build())
        cfg, buf, art, eff = C.POINTER(A.AgxHp1Config), C.POINTER(A.AgxHp1Buffers), C.POINTER(A.AgxArticulation), C.POINTER(A.AgxJointEffort)
        i, f, v = C.c_int, C.c_float, C.c_void_p
        argtypes = {
            "shadow_art_step": [cfg, buf, art],
            "shadow_art_step_imu": [cfg, buf, art, i, v],
            "shadow_art_step_effort": [cfg, buf, art, eff, i, v],
            "shadow_art_step_joint_force": [cfg, buf, art, eff, i, v, v, v],
            "shadow_art_body_state": [art, i, v, i, v],
            "shadow_art_dynamics": [art] + [v] * 5 + [f, v, i] + [v] * 5,
        }
        for name, args in argtypes.items():
            fn = getattr(lib, name)
            fn.argtypes = args
            fn.restype = None if name == "shadow_art_dynamics" else C.c_int
        _lib = lib
    return _lib


def body_state(art, root_state, body_state_out):
    """the shadow on torch CPU tensors: art = AgxArticulation (its dof_state pointer set), root_state [N,>=13] with contiguous rows,
    body_state_out [N,B,13] contiguous"""
    assert root_state.stride(1) == 1 and body_state_out.is_contiguous()
    rc = load().shadow_art_body_state(C.byref(art), root_state.shape[0], root_state.data_ptr(), root_state.stride(0),
                                      body_state_out.data_ptr())
    assert rc == 0
