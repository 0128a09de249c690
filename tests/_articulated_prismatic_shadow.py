"""Build + load the CPU shadow of the prismatic-joint kernels (tests/csrc/articulated_prismatic_shadow.cu).  Test infrastructure
only; built like tests/_articulated_shadow.py's library, with no FMA contraction."""
import ctypes as C
import os
import subprocess

from . import _articulated_shadow as S

SRC = os.path.join(S.HERE, "csrc", "articulated_prismatic_shadow.cu")
LIB = os.path.join(S.HERE, "_build", "libagx_articulated_prismatic_shadow.so")
_DEPS = [SRC] + S._DEPS[1:]
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
        raise RuntimeError("articulated prismatic shadow build failed:\n" + r.stdout + r.stderr)
    os.replace(tmp, LIB)
    return LIB


def load():
    global _lib
    if _lib is None:
        from aerial_gym_simulator_b200 import _lib as A
        lib = C.CDLL(build())
        cfg, buf, art, eff = C.POINTER(A.AgxHp1Config), C.POINTER(A.AgxHp1Buffers), C.POINTER(A.AgxArticulation), C.POINTER(A.AgxJointEffort)
        i, u, v = C.c_int, C.c_uint32, C.c_void_p
        for name, args in (("shadow_art_step_prismatic", [cfg, buf, art, u, eff, i, v, v, v]),
                           ("shadow_art_body_state_prismatic", [art, u, i, v, i, v])):
            fn = getattr(lib, name)
            fn.argtypes, fn.restype = args, C.c_int
        _lib = lib
    return _lib


def body_state(art, root_state, body_state_out, prismatic_mask):
    """the shadow of agx_hp1_articulated_body_state_prismatic on torch CPU tensors: art = AgxArticulation (its dof_state pointer
    set), root_state [N,>=13] with contiguous rows, body_state_out [N,B,13] contiguous"""
    assert root_state.stride(1) == 1 and body_state_out.is_contiguous()
    rc = load().shadow_art_body_state_prismatic(C.byref(art), prismatic_mask, root_state.shape[0], root_state.data_ptr(),
                                                root_state.stride(0), body_state_out.data_ptr())
    assert rc == 0
