"""CPU twin of an articulated robot's engine with joint force sensing, on top of tests/_cpu_stack_articulated_effort.py.  TEST
INFRASTRUCTURE ONLY.

``CpuJointForceHp1Engine`` is ``CpuEffortHp1Engine`` that also takes ``joint_force=`` (``joint_wrench`` / ``dof_force`` set up by
the PRODUCT's own ``Hp1Engine._init_joint_force``) and then steps on the host shadow of art_env_step<M, NB, true, true, true>
(tests/csrc/articulated_joint_force_shadow.cu), with the IMU input and the effort DOFs if the robot has them.  Without it it is
``CpuEffortHp1Engine``.

``with joint_force_cpu_stack():`` is ``cpu_stack()`` with EnvManager's engine swapped for this twin; ``joint_force_twin_for_dryrun()``
does the same swap inside the ``--gpu-dryrun`` fixture's ``cpu_stack()``."""
import contextlib
import ctypes as C

from aerial_gym_simulator_b200.hp1 import Hp1Engine

from . import _articulated_joint_force_shadow
from ._cpu_stack import cpu_stack
from ._cpu_stack_articulated_effort import CpuEffortHp1Engine


class CpuJointForceHp1Engine(CpuEffortHp1Engine):
    def __init__(self, spec, num_envs, device="cpu", *, joint_force=False, **kw):
        super().__init__(spec, num_envs, device, **kw)
        Hp1Engine._init_joint_force(self, joint_force)

    def physics_step(self, actions, disturbance=None, physics_steps=None, dist_counter=None, dist_offset=0):
        if self.joint_wrench is None:
            super().physics_step(actions, disturbance, physics_steps, dist_counter, dist_offset)
            return
        self._set_inputs(actions.contiguous(), disturbance, physics_steps, dist_counter, dist_offset)
        imu = self.imu_input is not None
        rc = _articulated_joint_force_shadow.load().shadow_art_step_joint_force(
            C.byref(self.cfg), C.byref(self._buf), C.byref(self.art), C.byref(self._effort) if self._effort is not None else None,
            self.imu_body if imu else 0, self.imu_input.data_ptr() if imu else None, self.joint_wrench.data_ptr(),
            self.dof_force.data_ptr() if self.dof_force.numel() else None)
        assert rc == 0


@contextlib.contextmanager
def _engine_swapped():
    import aerial_gym_simulator_b200.env_manager.env_manager as EM
    saved = EM.Hp1Engine
    EM.Hp1Engine = CpuJointForceHp1Engine
    try:
        yield
    finally:
        EM.Hp1Engine = saved


@contextlib.contextmanager
def joint_force_cpu_stack():
    with cpu_stack() as proxy, _engine_swapped():
        yield proxy


def joint_force_twin_for_dryrun():
    """inside the --gpu-dryrun fixture's cpu_stack(): EnvManager's engine becomes this twin (a context manager)"""
    return _engine_swapped()
