"""CPU twin of an articulated robot's engine with an IMU on one body, on top of tests/_cpu_stack_body_state.py.  TEST INFRASTRUCTURE
ONLY.

``CpuImuHp1Engine`` is ``CpuBodyStateHp1Engine`` that also takes ``imu_body=`` (``imu_input`` set up by the PRODUCT's own
``Hp1Engine._init_imu``) and then steps on the host shadow of art_env_step<M, NB, true> (tests/csrc/articulated_imu_shadow.cu).
Without ``imu_body`` it is ``CpuBodyStateHp1Engine``.

``with imu_cpu_stack():`` is ``cpu_stack()`` with EnvManager's engine swapped for this twin; ``imu_twin_for_dryrun()`` does the same
swap inside the ``--gpu-dryrun`` fixture's ``cpu_stack()``."""
import contextlib
import ctypes as C

from aerial_gym_simulator_b200.hp1 import Hp1Engine

from . import _articulated_imu_shadow
from ._cpu_stack import cpu_stack
from ._cpu_stack_body_state import CpuBodyStateHp1Engine


class CpuImuHp1Engine(CpuBodyStateHp1Engine):
    def __init__(self, spec, num_envs, device="cpu", *, imu_body=None, **kw):
        super().__init__(spec, num_envs, device, **kw)
        Hp1Engine._init_imu(self, imu_body)

    def physics_step(self, actions, disturbance=None, physics_steps=None, dist_counter=None, dist_offset=0):
        if self.imu_input is None:
            super().physics_step(actions, disturbance, physics_steps, dist_counter, dist_offset)
            return
        self._set_inputs(actions.contiguous(), disturbance, physics_steps, dist_counter, dist_offset)
        rc = _articulated_imu_shadow.load().shadow_art_step_imu(C.byref(self.cfg), C.byref(self._buf), C.byref(self.art), self.imu_body,
                                                                self.imu_input.data_ptr())
        assert rc == 0


@contextlib.contextmanager
def _engine_swapped():
    import aerial_gym_simulator_b200.env_manager.env_manager as EM
    saved = EM.Hp1Engine
    EM.Hp1Engine = CpuImuHp1Engine
    try:
        yield
    finally:
        EM.Hp1Engine = saved


@contextlib.contextmanager
def imu_cpu_stack():
    with cpu_stack() as proxy, _engine_swapped():
        yield proxy


def imu_twin_for_dryrun():
    """inside the --gpu-dryrun fixture's cpu_stack(): EnvManager's engine becomes this twin (a context manager)"""
    return _engine_swapped()
