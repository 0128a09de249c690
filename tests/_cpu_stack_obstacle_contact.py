"""CPU twins of the obstacle solves of EnvManager's sub-step, for an end-to-end dynamic_env run on the CPU stack.  Test
infrastructure only.  ``obstacle_twins()`` replaces, in env_manager, obstacle_obstacle_contact and obstacle_ground_contact by their
host shadows (the same contact_core.cuh text), the obstacle advance by agx_obstacle_step's host shadow, and the robot's contact
solve, which has no CPU twin (its contact search is the ray-caster's BVH), by a recorder.  None of them calls the library, so on a
machine with a GPU no kernel is launched on host memory.  Every call is logged in order, so a test sees the sub-step's sequence."""
import contextlib
import ctypes as C

import numpy as np

from tests import _contact_ground_shadow, _contact_obstacle_shadow, _shadow

_p = lambda a: C.c_void_p(a.ctypes.data)


def obstacle_obstacle_shadow(P, rows, mass, boxes, asset_box):
    """one launch of agx_obstacle_obstacle_contact on numpy arrays rows [E,A,>=13] (in place), mass [E,A,13], boxes [F,15],
    asset_box [E,A] -> (count [E], contacts [E,AGX_OBSTACLE_MAX_CONTACTS,9])"""
    E, A, stride = rows.shape
    assert rows.dtype == np.float32 and rows.flags.c_contiguous
    count = np.zeros(E, np.int32)
    contacts = np.zeros((E, 128, 9), np.float32)
    keep = [np.ascontiguousarray(mass, np.float32), np.ascontiguousarray(boxes, np.float32), np.ascontiguousarray(asset_box, np.int32)]
    _contact_obstacle_shadow.load().shadow_obstacle_obstacle(E, A, C.byref(P), _p(rows), stride, *(_p(x) for x in keep), _p(count),
                                                             _p(contacts))
    return count, contacts


def ground_shadow(P, rows, mass, hull):
    """one launch of agx_obstacle_ground_contact on numpy rows [E,A,>=13] (in place) with the hull of an ObstacleHull"""
    E, A, stride = rows.shape
    keep = [mass, hull.vertices.numpy(), hull.file_offset.numpy(), hull.file_reach.numpy(), hull.asset_file.numpy(),
            np.zeros((E * A, 8), np.int32), np.zeros(E * A, np.int32)]
    _contact_ground_shadow.load().shadow_obstacle_ground(E * A, C.byref(P), _p(rows), stride, *(_p(x) for x in keep))


@contextlib.contextmanager
def obstacle_twins():
    import aerial_gym_simulator_b200.env_manager.env_manager as EM

    log = []

    def pairs(params, motion, mass, boxes):
        st = motion.asset_state.numpy()
        obstacle_obstacle_shadow(params, st, mass.table.numpy(), boxes.boxes.numpy(), boxes.asset_file.numpy())
        log.append("obstacle_obstacle")

    def ground(params, motion, mass, hull):
        st = motion.asset_state.numpy()
        ground_shadow(params, st, mass.table.numpy(), hull)
        log.append("obstacle_ground")

    def robot(*args, **kw):
        log.append("robot_contact")

    def advance(self, twist, n):  # agx_obstacle_step's host shadow alone: nothing is launched on the device with host pointers
        ast = self.global_tensor_dict["env_asset_state_tensor"]
        twist = twist.contiguous() if twist is not None else None
        _shadow.load().shadow_obstacle_step(self.num_envs, self.num_obs_in_env, C.c_void_p(ast.data_ptr()), ast.stride(1),
                                            C.c_void_p(twist.data_ptr()) if twist is not None else None,
                                            float(self.sim_config.sim.dt), int(n), self._asset_damping[0], self._asset_damping[1])

    real_repose = EM.EnvManager._repose_scene

    def repose(self):
        log.append("repose")
        real_repose(self)

    saved = (EM.obstacle_obstacle_contact, EM.obstacle_ground_contact, EM.hp2_contact, EM.EnvManager._repose_scene,
             EM.EnvManager._advance_obstacles)
    (EM.obstacle_obstacle_contact, EM.obstacle_ground_contact, EM.hp2_contact, EM.EnvManager._repose_scene,
     EM.EnvManager._advance_obstacles) = pairs, ground, robot, repose, advance
    try:
        yield log
    finally:
        (EM.obstacle_obstacle_contact, EM.obstacle_ground_contact, EM.hp2_contact, EM.EnvManager._repose_scene,
         EM.EnvManager._advance_obstacles) = saved
