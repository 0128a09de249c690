"""CPU twin of an articulated robot's engine with effort-mode joints, on top of tests/_cpu_stack_articulated_imu.py.  TEST
INFRASTRUCTURE ONLY.

``CpuEffortHp1Engine`` is ``CpuImuHp1Engine`` whose ``dof_actuation_force`` and AgxJointEffort are set up by the PRODUCT's own
``Hp1Engine._init_effort``; a robot with an effort DOF then steps on the host shadow of art_env_step<M, NB, IMU, true>
(tests/csrc/articulated_effort_shadow.cu).  Without one it is ``CpuImuHp1Engine``.

``with effort_cpu_stack():`` is ``cpu_stack()`` with EnvManager's engine swapped for this twin; ``effort_twin_for_dryrun()`` does the
same swap inside the ``--gpu-dryrun`` fixture's ``cpu_stack()``."""
import contextlib
import ctypes as C

from aerial_gym_simulator_b200.hp1 import Hp1Engine

from . import _articulated_effort_shadow
from ._cpu_stack import cpu_stack
from ._cpu_stack_articulated_imu import CpuImuHp1Engine


class CpuEffortHp1Engine(CpuImuHp1Engine):
    def __init__(self, spec, num_envs, device="cpu", **kw):
        super().__init__(spec, num_envs, device, **kw)
        Hp1Engine._init_effort(self)

    def physics_step(self, actions, disturbance=None, physics_steps=None, dist_counter=None, dist_offset=0):
        if self._effort is None:
            super().physics_step(actions, disturbance, physics_steps, dist_counter, dist_offset)
            return
        self._set_inputs(actions.contiguous(), disturbance, physics_steps, dist_counter, dist_offset)
        imu = self.imu_input is not None
        rc = _articulated_effort_shadow.load().shadow_art_step_effort(C.byref(self.cfg), C.byref(self._buf), C.byref(self.art),
                                                                      C.byref(self._effort), self.imu_body if imu else 0,
                                                                      self.imu_input.data_ptr() if imu else None)
        assert rc == 0


@contextlib.contextmanager
def _engine_swapped():
    import aerial_gym_simulator_b200.env_manager.env_manager as EM
    saved = EM.Hp1Engine
    EM.Hp1Engine = CpuEffortHp1Engine
    try:
        yield
    finally:
        EM.Hp1Engine = saved


@contextlib.contextmanager
def effort_cpu_stack():
    with cpu_stack() as proxy, _engine_swapped():
        yield proxy


def effort_twin_for_dryrun():
    """inside the --gpu-dryrun fixture's cpu_stack(): EnvManager's engine becomes this twin (a context manager)"""
    return _engine_swapped()
