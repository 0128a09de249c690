"""CPU twin of an articulated robot's engine with prismatic joints, on top of tests/_cpu_stack_articulated.py.  TEST INFRASTRUCTURE ONLY.

``CpuPrismaticHp1Engine`` is ``CpuArticulatedHp1Engine`` for a robot with a prismatic joint: ``physics_step`` runs the host shadow
(tests/csrc/articulated_prismatic_shadow.cu) of the entry the PRODUCT's ``Hp1Engine._art_step_args`` picks,
agx_hp1_articulated_step_prismatic -> shadow_art_step_prismatic, with the same arguments, and ``update_body_state`` the shadow of
agx_hp1_articulated_body_state_prismatic.  Without a prismatic joint it is ``CpuArticulatedHp1Engine``.

``with prismatic_cpu_stack():`` is ``articulated_cpu_stack()`` with EnvManager's engine swapped for this twin;
``prismatic_twin_for_dryrun()`` does the same swap inside the ``--gpu-dryrun`` fixture's ``cpu_stack()``."""
import contextlib

from . import _articulated_prismatic_shadow
from ._cpu_stack import cpu_stack
from ._cpu_stack_articulated import CpuArticulatedHp1Engine


class CpuPrismaticHp1Engine(CpuArticulatedHp1Engine):
    def physics_step(self, actions, disturbance=None, physics_steps=None, dist_counter=None, dist_offset=0):
        if self.art is None or not self._prismatic:
            super().physics_step(actions, disturbance, physics_steps, dist_counter, dist_offset)
            return
        self._set_inputs(actions.contiguous(), disturbance, physics_steps, dist_counter, dist_offset)
        name, args = self._art_step_args()
        assert name == "agx_hp1_articulated_step_prismatic", name
        assert _articulated_prismatic_shadow.load().shadow_art_step_prismatic(*args) == 0

    def update_body_state(self):
        if self.art is None or not self._prismatic:
            super().update_body_state()
            return
        _articulated_prismatic_shadow.body_state(self.art, self.root_state, self.body_state, self._prismatic)


@contextlib.contextmanager
def _engine_swapped():
    import aerial_gym_simulator_b200.env_manager.env_manager as EM
    saved = EM.Hp1Engine
    EM.Hp1Engine = CpuPrismaticHp1Engine
    try:
        yield
    finally:
        EM.Hp1Engine = saved


@contextlib.contextmanager
def prismatic_cpu_stack():
    with cpu_stack() as proxy, _engine_swapped():
        yield proxy


def prismatic_twin_for_dryrun():
    """inside the --gpu-dryrun fixture's cpu_stack(): EnvManager's engine becomes the prismatic twin (a context manager)"""
    return _engine_swapped()
