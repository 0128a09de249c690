"""IMUSensor (sensors/imu_sensor.py:13-151): same surface -- init_tensors / update / reset / reset_idx, the
measurement lives in global_tensor_dict["imu_measurement"] -- with update() as ONE C-ABI call
(agx_imu_update).  Random numbers are drawn with torch in the reference's call order (randn for the
noise, randn for the bias walk; rand for resets).

`force_sensor_tensor` is PhysX's force-sensor reading in the reference (robot_manager.py:259-262, not
observable here): the total force on the link, gravity included, in the link frame.  EnvManager fills
it from the integrator: applied base-frame force of the last physics step (Hp1Engine body_wrench)
+ m R(q)^T g, so a hovering robot reads zero total force and the IMU reports +g along body z.

An IMU on a link (imu_config.parent_link): ``link_quat`` is the link's orientation in its body's frame, and the kernel reads
``mount_quats`` = link_quat (x) sensor_quats, refolded after every draw of sensor_quats (which stays relative to the link).
Without a link, ``mount_quats`` is ``sensor_quats`` itself."""
import ctypes as C
import math

import torch

from .. import _lib
from ..utils.math import quat_from_euler_xyz_tensor, quat_mul, torch_rand_float_tensor


class IMUSensor:
    def __init__(self, sensor_config, num_envs, device):
        self.cfg, self.num_envs, self.device = sensor_config, int(num_envs), torch.device(device)
        if self.device.type != "cuda":
            raise _lib.AgxError("IMUSensor needs a CUDA device: there is no CPU path")
        self.lib = _lib.load()
        self.world_frame = self.cfg.world_frame
        self.gravity_compensation = self.cfg.gravity_compensation

    def init_tensors(self, global_tensor_dict=None):
        gtd, N, dev = global_tensor_dict, self.num_envs, self.device
        self.global_tensor_dict = gtd
        self.robot_state = gtd["robot_state_tensor"]  # orientation = columns 3..6 (IGE_env_manager.py:301-311)
        self.robot_body_angvel = gtd["robot_body_angvel"]
        self.robot_masses = gtd["robot_mass"].contiguous()
        self.force_sensor_tensor = gtd["force_sensor_tensor"]
        self.dt = gtd["dt"]
        self.sqrt_dt = math.sqrt(self.dt)
        T = lambda v: torch.tensor(v, dtype=torch.float32, device=dev)
        self.max_bias_init_value = T(self.cfg.max_bias_init_value)
        self.min_sensor_euler_rotation_rad = torch.deg2rad(T(self.cfg.min_euler_rotation_deg)).expand(N, -1)
        self.max_sensor_euler_rotation_rad = torch.deg2rad(T(self.cfg.max_euler_rotation_deg)).expand(N, -1)
        self.sensor_quats = quat_from_euler_xyz_tensor(
            torch_rand_float_tensor(self.min_sensor_euler_rotation_rad, self.max_sensor_euler_rotation_rad)).contiguous()
        self.link_quat, self.mount_quats = None, self.sensor_quats
        self.bias = torch.zeros(N, 6, device=dev)
        self.imu_meas = torch.zeros(N, 6, device=dev)
        gtd["imu_measurement"] = self.imu_meas
        c = _lib.AgxImuConfig()
        c.world_frame, c.enable_noise, c.enable_bias = int(self.world_frame), int(self.cfg.enable_noise), int(self.cfg.enable_bias)
        c.sqrt_dt = self.sqrt_dt
        g = gtd["gravity"][0].tolist() if torch.is_tensor(gtd["gravity"]) else list(gtd["gravity"])
        for i in range(3):
            c.g_world[i] = g[i] * (1 - int(self.gravity_compensation))  # imu_sensor.py:61-63
        for i in range(6):
            c.bias_std[i], c.noise_std[i], c.max_meas[i] = self.cfg.bias_std[i], self.cfg.imu_noise_std[i], self.cfg.max_measurement_value[i]
        self._c = c

    def update(self, n_noise=None, n_bias=None):
        """n_noise / n_bias: optional explicit standard-normal draws [N,6] (tests); default torch.randn in the
        reference's order (sample_noise, then update_bias)."""
        N, dev = self.num_envs, self.device
        if n_noise is None:
            n_noise = torch.randn((N, 6), device=dev)
        if n_bias is None:
            n_bias = torch.randn((N, 6), device=dev)
        f, st = self.force_sensor_tensor, self.robot_state
        if f.stride(-1) != 1 or st.stride(-1) != 1:
            raise ValueError("force_sensor_tensor / robot_state_tensor rows must be contiguous")
        p = lambda t: C.c_void_p(t.data_ptr())
        _lib.check(self.lib.agx_imu_update(N, C.byref(self._c), p(f), f.stride(0), p(self.robot_masses), p(st), st.stride(0),
                                           p(self.robot_body_angvel), p(self.mount_quats), p(n_noise), p(n_bias), p(self.bias),
                                           p(self.imu_meas), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)), "agx_imu_update")

    def set_link(self, link_quat):
        """mount the IMU on a link whose frame is rotated by link_quat [4] (xyzw) in the frame of the body the kernel reads"""
        self.link_quat = link_quat.to(self.device, torch.float32)
        self.mount_quats = torch.zeros_like(self.sensor_quats)
        self._fold_link()

    def _fold_link(self):
        if self.link_quat is None:
            return
        self.mount_quats.copy_(quat_mul(self.link_quat.expand_as(self.sensor_quats), self.sensor_quats))

    def reset(self):
        self.bias[:] = self.max_bias_init_value * (2.0 * (torch.rand_like(self.bias) - 0.5))
        self.sensor_quats[:] = quat_from_euler_xyz_tensor(
            torch_rand_float_tensor(self.min_sensor_euler_rotation_rad, self.max_sensor_euler_rotation_rad))
        self._fold_link()

    def reset_idx(self, env_ids):
        self.bias[env_ids, :] = (self.max_bias_init_value * (2.0 * (torch.rand_like(self.bias) - 0.5)))[env_ids, :]
        self.sensor_quats[env_ids] = quat_from_euler_xyz_tensor(
            torch_rand_float_tensor(self.min_sensor_euler_rotation_rad, self.max_sensor_euler_rotation_rad))[env_ids]
        self._fold_link()

    def get_observation(self):
        return self.imu_meas
