"""ctypes binding of libaerial_gym_b200.so (the C ABI in include/aerial_gym_b200.h).

Fails loudly: no library -> ImportError-like RuntimeError naming the build command;
nothing here falls back to torch or CPU code."""
import ctypes as C
import os

from . import _build

AGX_MAX_MOTORS = 8

# controller ids (AGX_CTRL_*)
CTRL_NONE, CTRL_ATTITUDE, CTRL_POSITION, CTRL_VELOCITY = 0, 1, 2, 3
CTRL_ACCELERATION, CTRL_RATES, CTRL_FULLY_ACTUATED, CTRL_VELOCITY_STEERING = 4, 5, 6, 7
# flags (AGX_F_*)
F_USE_RPS, F_MOTOR_RK4, F_DISCRETE_MIX, F_GYROSCOPIC = 0x1, 0x2, 0x4, 0x8
F_RANDOMIZE_GAINS, F_DEVICE_RNG_RESET, F_STRICT_STALE_OBS = 0x10, 0x20, 0x40

f32 = C.c_float
fp = C.c_void_p  # device pointers travel as integers


class AgxHp1Config(C.Structure):
    _fields_ = [
        ("num_envs", C.c_int32), ("num_motors", C.c_int32), ("controller", C.c_int32),
        ("num_actions", C.c_int32), ("physics_steps", C.c_int32), ("flags", C.c_int32),
        ("episode_len_steps", C.c_int32), ("env_id_offset", C.c_int32),
        ("seed", C.c_uint64),
        ("dt", f32), ("gravity", f32 * 3), ("mass", f32),
        ("inertia", f32 * 9), ("inertia_inv", f32 * 9),
        ("alloc_pinv", f32 * (AGX_MAX_MOTORS * 6)), ("wrench_map", f32 * (6 * AGX_MAX_MOTORS)),
        ("com", f32 * 3),
        ("min_thrust", f32), ("max_thrust", f32), ("max_thrust_rate", f32), ("max_yaw_rate", f32),
        ("drag_lin1", f32 * 3), ("drag_lin2", f32 * 3), ("drag_ang1", f32 * 3), ("drag_ang2", f32 * 3),
        ("linear_damping", f32), ("angular_damping", f32),
        ("max_linear_velocity", f32), ("max_angular_velocity", f32),
        ("K_pos", f32 * 3), ("K_vel", f32 * 3), ("K_rot", f32 * 3), ("K_angvel", f32 * 3),
        ("tau_inc", f32), ("tau_dec", f32), ("k_thrust", f32), ("crash_distance", f32),
        ("min_init_state", f32 * 13), ("max_init_state", f32 * 13),
        ("bounds_lo_min", f32 * 3), ("bounds_lo_max", f32 * 3),
        ("bounds_hi_min", f32 * 3), ("bounds_hi_max", f32 * 3),
        ("tau_inc_range", f32 * 2), ("tau_dec_range", f32 * 2), ("k_thrust_range", f32 * 2),
        ("K_pos_min", f32 * 3), ("K_pos_max", f32 * 3), ("K_vel_min", f32 * 3), ("K_vel_max", f32 * 3),
        ("K_rot_min", f32 * 3), ("K_rot_max", f32 * 3), ("K_angvel_min", f32 * 3), ("K_angvel_max", f32 * 3),
        ("dist_prob", f32), ("dist_max", f32 * 6), ("dist_pad_", C.c_uint32), ("dist_seed", C.c_uint64),
    ]


_HP1_BUF_FIELDS = [
    "root_state", "motor_thrust", "sim_steps", "actions", "disturbance", "dist_counter", "dist_offset_", "target_position",
    "tau_inc", "tau_dec", "k_thrust", "K_pos", "K_vel", "K_rot", "K_angvel", "bounds_min", "bounds_max",
    "euler", "vehicle_orientation", "vehicle_linvel", "body_linvel", "body_angvel", "body_wrench",
    "obs", "reward", "terminations", "truncations", "reset_mask", "any_reset", "episode_count", "fresh_vel", "publish_ctr", "tile_sync",
]


class AgxHp1Buffers(C.Structure):
    # dist_offset_: the uint32 pair (dist_offset, pad) travels as one 8-byte slot; the `dist_offset` property reads / writes its low word
    _fields_ = [(n, (C.c_uint64 if n == "dist_offset_" else fp)) for n in _HP1_BUF_FIELDS]

    @property
    def dist_offset(self):
        return self.dist_offset_ & 0xFFFFFFFF

    @dist_offset.setter
    def dist_offset(self, v):
        self.dist_offset_ = int(v) & 0xFFFFFFFF


class AgxObsGatherPush(C.Structure):
    _fields_ = [("local", fp), ("peer_bufs", fp), ("peer_flags", fp), ("world", C.c_int32), ("rank", C.c_int32),
                ("bytes", C.c_uint64), ("epoch", C.c_uint32), ("max_ctas", C.c_int32), ("ready_ctr", fp), ("ready_target", C.c_uint64),
                ("scratch", fp), ("error_word", fp), ("flag_slot", C.c_int32), ("pad_", C.c_int32), ("read_done", fp), ("mc_buf", fp)]


_HP1_DRAW_FIELDS = ["bounds_lo", "bounds_hi", "state", "K_pos", "K_vel", "K_rot", "K_angvel",
                    "tau_inc", "tau_dec", "thrust", "k_thrust"]


class AgxHp1ResetDraws(C.Structure):
    _fields_ = [(n, fp) for n in _HP1_DRAW_FIELDS]


class AgxNavRewardParams(C.Structure):
    _fields_ = [("v", C.c_float * 18)]


class AgxLidarNavRewardParams(C.Structure):
    _fields_ = [("v", C.c_float * 22), ("radar_variant", C.c_int32)]


class AgxE2ERewardParams(C.Structure):
    _fields_ = [(n, C.c_float) for n in ("z_error_scale", "upright_gain2", "upright_exp2", "align_gain1", "align_exp1", "align_gain2",
                                         "align_exp2", "angvel_gain", "hover_thrust", "towards_gain_pos", "towards_gain_neg",
                                         "action_diff_gain", "crash_dist")]


class AgxImuConfig(C.Structure):
    _fields_ = [("world_frame", C.c_int32), ("enable_noise", C.c_int32), ("enable_bias", C.c_int32), ("sqrt_dt", C.c_float),
                ("g_world", C.c_float * 3), ("bias_std", C.c_float * 6), ("noise_std", C.c_float * 6), ("max_meas", C.c_float * 6)]


class AgxHp2Scene(C.Structure):
    _fields_ = [
        ("num_envs", C.c_int32), ("num_objects", C.c_int32), ("leaves_pow2", C.c_int32),
        ("tris_per_object", C.c_int32), ("num_templates", C.c_int32), ("obj_pose_stride", C.c_int32),
        ("tmpl_tri_offset", fp), ("tmpl_tris", fp), ("tmpl_seg_base", fp), ("tmpl_seg_mask", fp),
        ("obj_pose", fp), ("obj_template", fp), ("obj_seg_counter", fp), ("bounds_min", fp), ("bounds_max", fp),
        ("tris", fp), ("nodes", fp), ("leaf_object", fp), ("face_offset", fp), ("tmpl_obb", fp), ("obb", fp),
    ]


class AgxHp2Sensor(C.Structure):
    _fields_ = [
        ("kind", C.c_int32), ("width", C.c_int32), ("height", C.c_int32), ("num_sensors", C.c_int32),
        ("calculate_depth", C.c_int32), ("return_pointcloud", C.c_int32), ("pointcloud_in_world_frame", C.c_int32),
        ("segmentation", C.c_int32), ("fuse_epilogue", C.c_int32), ("normalize_range", C.c_int32),
        ("c_x", C.c_int32), ("c_y", C.c_int32), ("kinv", f32 * 9), ("far_plane", f32),
        ("max_range", f32), ("min_range", f32), ("far_out_of_range_value", f32), ("near_out_of_range_value", f32),
        ("frame_quat", f32 * 4), ("baseline", f32), ("normal_in_world_frame", C.c_int32),
        ("robot_pose_stride", C.c_int32), ("pad_", C.c_int32),
        ("robot_pose", fp), ("mount", fp), ("ray_table", fp), ("pixels", fp), ("seg_pixels", fp),
    ]


class AgxHp2Noise(C.Structure):
    _fields_ = [("components", C.c_int32), ("enable_noise", C.c_int32), ("apply_limits", C.c_int32), ("normalize", C.c_int32),
                ("std_a", f32), ("std_b", f32), ("std_c", f32), ("mean_offset", f32), ("pixel_dropout_prob", f32),
                ("max_range", f32), ("min_range", f32), ("far_out_of_range_value", f32), ("near_out_of_range_value", f32)]


SENSOR_CAMERA, SENSOR_LIDAR, SENSOR_STEREO_CAMERA, SENSOR_NORMAL_FACEID_CAMERA, SENSOR_NORMAL_FACEID_LIDAR = 0, 1, 2, 3, 4


class AgxError(RuntimeError):
    pass


_lib = None


def lib_path():
    # AGX_LIB_PATH: A/B experiments against an alternative build of the same ABI
    return os.environ.get("AGX_LIB_PATH", _build.LIB)


def load():
    """Load (once) and type the library.  Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    path = lib_path()
    if not os.path.exists(path):
        raise AgxError(
            f"{path} not found: build it with `python -m aerial_gym_simulator_b200._build` "
            "(nvcc, sm_90a).  There is no CPU / torch fallback."
        )
    lib = C.CDLL(path)
    lib.agx_abi_version.restype = C.c_int
    lib.agx_last_error.restype = C.c_char_p
    lib.agx_sizeof.restype = C.c_uint64
    lib.agx_sizeof.argtypes = [C.c_int]
    for name, args in {
        "agx_hp1_physics_step": [C.POINTER(AgxHp1Config), C.POINTER(AgxHp1Buffers), C.c_void_p],
        "agx_hp1_position_task_step": [C.POINTER(AgxHp1Config), C.POINTER(AgxHp1Buffers), C.c_void_p],
        "agx_hp1_position_task_step_profiled": [C.POINTER(AgxHp1Config), C.POINTER(AgxHp1Buffers), C.c_void_p,
                                                C.c_void_p],
        "agx_hp1_reset": [C.POINTER(AgxHp1Config), C.POINTER(AgxHp1Buffers), C.c_void_p,
                          C.POINTER(AgxHp1ResetDraws), C.c_void_p],
        "agx_hp1_refresh": [C.POINTER(AgxHp1Config), C.POINTER(AgxHp1Buffers), C.c_int, C.c_void_p],
        "agx_hp2_update_scene": [C.POINTER(AgxHp2Scene), C.c_void_p, C.c_void_p],
        "agx_hp2_cast": [C.POINTER(AgxHp2Scene), C.POINTER(AgxHp2Sensor), C.c_void_p],
        "agx_p2p_allgather": [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_uint64, C.c_uint32, C.c_void_p, C.c_void_p],
        "agx_obs_gather_push": [C.POINTER(AgxObsGatherPush), C.c_void_p],
        "agx_obs_gather_wait": [C.c_void_p, C.c_int, C.c_int, C.c_uint32, C.c_void_p, C.c_void_p],
        "agx_obs_gather_check": [C.c_void_p, C.c_void_p],
        "agx_obs_gather_gate": [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p],
        "agx_obs_gather_set_timeout_ns": [C.c_uint64],
        "agx_set_spin_timeout_ms": [C.c_uint64],
        "agx_hp1_check": [C.POINTER(AgxHp1Buffers), C.c_void_p],
        "agx_hp1_position_task_step_gathered": [C.POINTER(AgxHp1Config), C.POINTER(AgxHp1Buffers), C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p,
                                                C.POINTER(AgxObsGatherPush), C.c_void_p],
        "agx_counter_add": [C.c_void_p, C.c_uint32, C.c_void_p],
        "agx_hp1_task_step_is_chained": [C.POINTER(AgxHp1Config), C.POINTER(AgxHp1Buffers)],
        "agx_nav_reward": [C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float,
                           C.POINTER(AgxNavRewardParams), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p],
        "agx_nav_obs": [C.c_int, C.c_void_p, C.c_int] + [C.c_void_p] * 9 + [C.c_int, C.c_void_p],
        "agx_imu_update": [C.c_int, C.POINTER(AgxImuConfig), C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int] + [C.c_void_p] * 7,
        "agx_lidar_nav_pool": [C.c_int] * 5 + [C.c_void_p, C.c_void_p, C.c_int] + [C.c_float] * 4 + [C.c_void_p] * 3,
        "agx_lidar_nav_reward": [C.c_int, C.c_void_p, C.c_int] + [C.c_void_p] * 10 + [C.c_float, C.POINTER(AgxLidarNavRewardParams)]
                                + [C.c_void_p] * 4,
        "agx_lidar_nav_obs": [C.c_int, C.c_void_p, C.c_int] + [C.c_void_p] * 10 + [C.c_int, C.c_void_p, C.c_int, C.c_void_p],
        "agx_e2e_reward": [C.c_int, C.c_void_p, C.c_int] + [C.c_void_p] * 5 + [C.POINTER(AgxE2ERewardParams)] + [C.c_void_p] * 3,
        "agx_e2e_obs": [C.c_int, C.c_void_p, C.c_int] + [C.c_void_p] * 4 + [C.c_int, C.c_void_p],
        "agx_s2r_reward": [C.c_int, C.c_int, C.c_void_p, C.c_int] + [C.c_void_p] * 10,
        "agx_s2r_obs": [C.c_int, C.c_void_p, C.c_int] + [C.c_void_p] * 6 + [C.c_int, C.c_void_p],
        "agx_disturbance_draw": [C.c_int, C.c_int, C.c_float, C.POINTER(C.c_float), C.c_uint64, C.c_uint32, C.c_void_p, C.c_void_p],
        "agx_obstacle_step": [C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_float, C.c_int, C.c_float, C.c_float, C.c_void_p],
        "agx_hp2_noise_limits": [C.c_void_p, C.c_uint64, C.c_uint64, C.POINTER(AgxHp2Noise), C.c_uint64, C.c_uint32, C.c_void_p],
        "agx_host_alloc": [C.c_uint64, C.POINTER(C.c_void_p)],
        "agx_host_free": [C.c_void_p],
        "agx_hp2_collide": [C.POINTER(AgxHp2Scene), C.c_void_p, C.c_int, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p],
    }.items():
        try:
            fn = getattr(lib, name)
        except AttributeError:
            raise AgxError(f"{path} does not export {name}: it was built from older sources than include/aerial_gym_b200.h -- "
                           "rebuild it with `python -m aerial_gym_simulator_b200._build --force`") from None
        fn.restype = C.c_int
        fn.argtypes = args
    lib.agx_hp2_scene_bytes.restype = C.c_uint64
    lib.agx_hp2_scene_bytes.argtypes = [C.c_int, C.c_int, C.c_int]
    if lib.agx_sizeof(3) != C.sizeof(AgxHp2Scene) or lib.agx_sizeof(4) != C.sizeof(AgxHp2Sensor):
        raise AgxError("HP2 ABI struct size mismatch between _lib.py and libaerial_gym_b200.so")
    if lib.agx_sizeof(5) != C.sizeof(AgxNavRewardParams) or lib.agx_sizeof(6) != C.sizeof(AgxImuConfig) \
            or lib.agx_sizeof(7) != C.sizeof(AgxLidarNavRewardParams) or lib.agx_sizeof(8) != C.sizeof(AgxHp2Noise) \
            or lib.agx_sizeof(9) != C.sizeof(AgxE2ERewardParams):
        raise AgxError("aux ABI struct size mismatch between _lib.py and libaerial_gym_b200.so")
    if lib.agx_sizeof(0) != C.sizeof(AgxHp1Config) or lib.agx_sizeof(1) != C.sizeof(AgxHp1Buffers) \
            or lib.agx_sizeof(2) != C.sizeof(AgxHp1ResetDraws) or lib.agx_sizeof(10) != C.sizeof(AgxObsGatherPush):
        raise AgxError("ABI struct size mismatch between _lib.py and libaerial_gym_b200.so")
    _lib = lib
    return lib


def check(rc, what=""):
    if rc != 0:
        raise AgxError(f"{what} failed ({rc}): {load().agx_last_error().decode()}")


def declared_symbols():
    """extern "C" function names declared in include/aerial_gym_b200.h (for the export test)."""
    import re
    hdr = os.path.join(os.path.dirname(_build.PKG), "include", "aerial_gym_b200.h")
    txt = open(hdr).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(agx_[a-z0-9_]+)\s*\(", txt)))
