"""CPU twin of an articulated robot's engine, on top of tests/_cpu_stack.py.  TEST INFRASTRUCTURE ONLY.

``CpuArticulatedHp1Engine`` is ``CpuHp1Engine`` that also takes ``articulation=`` (an ArticulationSpec): the joint tensors and the
AgxArticulation struct are set up by the PRODUCT's own ``Hp1Engine._init_articulation`` (on CPU tensors), and ``physics_step`` of
an articulated robot runs the host shadow of articulated_core.cuh (tests/csrc/articulated_shadow.cu).  Without ``articulation`` it
is ``CpuHp1Engine``.

``with articulated_cpu_stack():`` is ``cpu_stack()`` with EnvManager's engine swapped for this twin, so an EnvManager (and a task)
with ``morphy_compliant`` runs end to end on the CPU.  ``articulated_twin_for_dryrun(module)`` does the same swap inside an already
entered ``cpu_stack()`` -- what the ``--gpu-dryrun`` fixture of tests/conftest.py enters for a -m gpu test."""
import contextlib
import ctypes as C

from aerial_gym_simulator_b200.hp1 import Hp1Engine

from . import _articulated_shadow
from ._cpu_stack import CpuHp1Engine, cpu_stack
from ._shadow_hp1 import ShadowHp1Engine


class CpuArticulatedHp1Engine(CpuHp1Engine):
    def __init__(self, spec, num_envs, device="cpu", *, articulation=None, debug_wrench=False, host_io=False, **kw):
        super().__init__(spec, num_envs, device, debug_wrench=debug_wrench, host_io=host_io, **kw)
        Hp1Engine._init_articulation(self, articulation, num_envs, debug_wrench, host_io)

    def position_task_step(self, actions, disturbance=None, physics_steps=None, mid_event=None):
        if self.art is not None:
            raise ValueError("an articulated robot has no fused task step: step it with physics_step (PositionSetpointTask does)")
        super().position_task_step(actions, disturbance, physics_steps, mid_event)

    def physics_step(self, actions, disturbance=None, physics_steps=None, dist_counter=None, dist_offset=0):
        if self.art is None:
            ShadowHp1Engine.physics_step(self, actions.contiguous(), disturbance, physics_steps, dist_counter, dist_offset)
            return
        self._set_inputs(actions.contiguous(), disturbance, physics_steps, dist_counter, dist_offset)
        assert _articulated_shadow.load().shadow_art_step(C.byref(self.cfg), C.byref(self._buf), C.byref(self.art)) == 0


@contextlib.contextmanager
def _engine_swapped():
    import aerial_gym_simulator_b200.env_manager.env_manager as EM
    saved = EM.Hp1Engine
    EM.Hp1Engine = CpuArticulatedHp1Engine
    try:
        yield
    finally:
        EM.Hp1Engine = saved


@contextlib.contextmanager
def articulated_cpu_stack():
    with cpu_stack() as proxy, _engine_swapped():
        yield proxy


def articulated_twin_for_dryrun():
    """inside the --gpu-dryrun fixture's cpu_stack(): EnvManager's engine becomes the articulated twin (a context manager)"""
    return _engine_swapped()
