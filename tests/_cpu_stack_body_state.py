"""CPU twin of an articulated robot's per-body state, on top of tests/_cpu_stack_articulated.py.  TEST INFRASTRUCTURE ONLY.

``CpuBodyStateHp1Engine`` is ``CpuArticulatedHp1Engine`` that also owns ``body_state`` (set up by the PRODUCT's own
``Hp1Engine._init_body_state``) and runs ``update_body_state`` on the host shadow of articulated_core.cuh's art_body_states
(tests/csrc/articulated_body_state_shadow.cu).

``with body_state_cpu_stack():`` is ``cpu_stack()`` with EnvManager's engine swapped for this twin; ``body_state_twin_for_dryrun()``
does the same swap inside the ``--gpu-dryrun`` fixture's ``cpu_stack()``."""
import contextlib
import ctypes as C
import os
import subprocess

from aerial_gym_simulator_b200.hp1 import Hp1Engine

from ._cpu_stack import cpu_stack
from ._cpu_stack_articulated import CpuArticulatedHp1Engine

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "csrc", "articulated_body_state_shadow.cu")
LIB = os.path.join(HERE, "_build", "libagx_articulated_body_state_shadow.so")
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
        raise RuntimeError("articulated body-state shadow build failed:\n" + r.stdout + r.stderr)
    os.replace(tmp, LIB)
    return LIB


def load():
    global _lib
    if _lib is None:
        from aerial_gym_simulator_b200 import _lib as A
        lib = C.CDLL(build())
        lib.shadow_art_body_state.restype = C.c_int
        lib.shadow_art_body_state.argtypes = [C.POINTER(A.AgxArticulation), C.c_int, C.c_void_p, C.c_int, C.c_void_p]
        _lib = lib
    return _lib


def body_state(art, root_state, body_state_out):
    """the shadow on torch CPU tensors: art = AgxArticulation (its dof_state pointer set), root_state [N,>=13] with contiguous rows,
    body_state_out [N,B,13] contiguous"""
    assert root_state.stride(1) == 1 and body_state_out.is_contiguous()
    rc = load().shadow_art_body_state(C.byref(art), root_state.shape[0], root_state.data_ptr(), root_state.stride(0),
                                      body_state_out.data_ptr())
    assert rc == 0


class CpuBodyStateHp1Engine(CpuArticulatedHp1Engine):
    def __init__(self, spec, num_envs, device="cpu", **kw):
        super().__init__(spec, num_envs, device, **kw)
        Hp1Engine._init_body_state(self)

    def update_body_state(self):
        if self.art is None:
            raise ValueError("body_state belongs to an articulated robot (Hp1Engine(articulation=...))")
        body_state(self.art, self.root_state, self.body_state)


@contextlib.contextmanager
def _engine_swapped():
    import aerial_gym_simulator_b200.env_manager.env_manager as EM
    saved = EM.Hp1Engine
    EM.Hp1Engine = CpuBodyStateHp1Engine
    try:
        yield
    finally:
        EM.Hp1Engine = saved


@contextlib.contextmanager
def body_state_cpu_stack():
    with cpu_stack() as proxy, _engine_swapped():
        yield proxy


def body_state_twin_for_dryrun():
    """inside the --gpu-dryrun fixture's cpu_stack(): EnvManager's engine becomes this twin (a context manager)"""
    return _engine_swapped()
