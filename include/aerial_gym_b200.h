/*
 * aerial_gym_b200 -- C ABI of the H100-native hot paths (libaerial_gym_b200.so).
 *
 * The reference (ntnu-arl/aerial_gym_simulator, commit f0d0f05) has NO plugin / FFI boundary
 * for these paths: they sit behind plain Python objects (SURVEY.md section 8b).  The entry
 * points below are therefore the narrowest C surface that replaces, one for one, the Python
 * call sites listed beside each function.  Conventions:
 *
 *   - plain C, POD structs, raw device pointers + sizes; no torch / C++ types;
 *   - the caller (PyTorch) owns every buffer; the library never allocates user-visible
 *     memory, never frees, never synchronises the stream unless the function says so;
 *   - every function returns 0 on success or a negative AGX_E_* code; agx_last_error()
 *     returns a thread-local message; no exceptions cross the boundary;
 *   - kernels are launched on the cudaStream_t passed in (as void*; 0 = legacy default).
 *
 * HP1 = rigid-body integrator + rotor/motor model + Lee controller + allocation.
 * HP2 = depth / segmentation / LiDAR ray-caster.
 */
#ifndef AERIAL_GYM_B200_H_
#define AERIAL_GYM_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define AGX_ABI_VERSION 1
#define AGX_MAX_MOTORS 8

/* error codes */
#define AGX_OK 0
#define AGX_E_INVALID (-1)   /* bad argument / unsupported configuration */
#define AGX_E_CUDA (-2)      /* CUDA runtime error (message in agx_last_error) */
#define AGX_E_NULL (-3)      /* required pointer is NULL */
#define AGX_E_TIMEOUT (-4)   /* a bounded in-kernel wait expired (agx_hp1_check / agx_obs_gather_check) */

/* controller ids -- one per reference controller class (aerial_gym/control/__init__.py:42-99) */
#define AGX_CTRL_NONE 0              /* NoControl                       controllers/no_control.py:29-30 */
#define AGX_CTRL_ATTITUDE 1          /* LeeAttitudeController           controllers/attitude_control.py:16-43 */
#define AGX_CTRL_POSITION 2          /* LeePositionController           controllers/position_control.py:21-51 */
#define AGX_CTRL_VELOCITY 3          /* LeeVelocityController           controllers/velocity_control.py:17-53 */
#define AGX_CTRL_ACCELERATION 4      /* LeeAccelerationController       controllers/acceleration_control.py:16-46 */
#define AGX_CTRL_RATES 5             /* LeeRatesController              controllers/rates_control.py:16-28 */
#define AGX_CTRL_FULLY_ACTUATED 6    /* FullyActuatedController         controllers/fully_actuated_control.py:14-32 */
#define AGX_CTRL_VELOCITY_STEERING 7 /* LeeVelocitySteeringAngleController controllers/velocity_steeing_angle_controller.py:16-50 */

/* AgxHp1Config.flags */
#define AGX_F_USE_RPS 0x1            /* motor_model.py:98 (cfg.use_rps) */
#define AGX_F_MOTOR_RK4 0x2          /* motor_model.py:13-19 (default rk4) */
#define AGX_F_DISCRETE_MIX 0x4       /* motor_model.py:201-210 */
#define AGX_F_GYROSCOPIC 0x8         /* integrator spec: include -W x JW */
#define AGX_F_RANDOMIZE_GAINS 0x10   /* base_lee_controller.py:101-118 (cfg.randomize_params) */
#define AGX_F_DEVICE_RNG_RESET 0x20  /* fused step resets finished envs in-kernel (Philox4x32-10) */
#define AGX_F_STRICT_STALE_OBS 0x40  /* reproduce the stale-derived-state quirk (SURVEY 3.1) */

typedef struct AgxHp1Config {
    int32_t num_envs;
    int32_t num_motors;        /* M in [1, AGX_MAX_MOTORS] */
    int32_t controller;        /* AGX_CTRL_* */
    int32_t num_actions;       /* columns of the action tensor */
    int32_t physics_steps;     /* physics steps per call (env_manager.py:417-428) */
    int32_t flags;             /* AGX_F_* */
    int32_t episode_len_steps; /* position task: truncation when sim_steps > this */
    int32_t env_id_offset;     /* global id of local env 0 (multi-GPU sharding; keys the device RNG) */
    uint64_t seed;             /* device RNG key */
    float dt;
    float gravity[3];
    float mass;
    float inertia[9];          /* row-major, about the COM, base frame */
    float inertia_inv[9];
    float alloc_pinv[AGX_MAX_MOTORS * 6]; /* [M][6] pinv(A), control_allocation.py:46-48 */
    float wrench_map[6 * AGX_MAX_MOTORS]; /* [6][M] motor thrust -> base-frame wrench about the COM */
    float com[3];
    float min_thrust, max_thrust, max_thrust_rate;
    float max_yaw_rate;
    float drag_lin1[3], drag_lin2[3], drag_ang1[3], drag_ang2[3]; /* base_multirotor.py:260-285 */
    float linear_damping, angular_damping;   /* base_quad_config.py:93-94 */
    float max_linear_velocity, max_angular_velocity;
    /* per-env parameter arrays may be NULL in AgxHp1Buffers; these constants are used instead */
    float K_pos[3], K_vel[3], K_rot[3], K_angvel[3];
    float tau_inc, tau_dec, k_thrust;
    float crash_distance;      /* position task: crash when |target - x| > this (8.0) */
    /* reset ranges (uniform: lo + (hi - lo) * u) */
    float min_init_state[13], max_init_state[13]; /* base_quad_config.py:30-59 */
    float bounds_lo_min[3], bounds_lo_max[3];     /* env_config/empty_env.py:27-31 */
    float bounds_hi_min[3], bounds_hi_max[3];
    float tau_inc_range[2], tau_dec_range[2], k_thrust_range[2];
    float K_pos_min[3], K_pos_max[3], K_vel_min[3], K_vel_max[3];
    float K_rot_min[3], K_rot_max[3], K_angvel_min[3], K_angvel_max[3];
    /* in-kernel disturbance (AgxHp1Buffers.dist_counter != NULL): BaseMultirotor.apply_disturbance (base_multirotor.py:213-234)
     * drawn inside the physics sub-step with the same Philox stream as agx_disturbance_draw (disturbance_core.cuh) */
    float dist_prob;
    float dist_max[6];
    uint32_t dist_pad_;
    uint64_t dist_seed;
} AgxHp1Config;

/* All pointers are DEVICE pointers.  [N,...] arrays are dense row-major fp32 unless noted. */
typedef struct AgxHp1Buffers {
    /* state (read + written) */
    float* root_state;        /* [N,13] x y z qx qy qz qw vx vy vz wx wy wz  (IGE_env_manager.py:347-358) */
    float* motor_thrust;      /* [N,M]  MotorModel.current_motor_thrust */
    int32_t* sim_steps;       /* [N]    env_manager.py:78-80 (may be NULL for agx_hp1_physics_step) */
    /* inputs */
    const float* actions;     /* [N,num_actions] */
    const float* disturbance; /* [N,6] gated body-0 wrench or NULL (base_multirotor.py:213-234) */
    const uint32_t* dist_counter; /* device u32 or NULL (agx_hp1_physics_step only).  When `disturbance` is NULL and this is set, physics sub-step s of the launch
                                     draws its disturbance in the kernel with draw counter *dist_counter + dist_offset + s -- bit for bit
                                     what agx_disturbance_draw(counter = that value) would have put into `disturbance`.  The counter
                                     lives in device memory so that a CUDA graph of an env step (n physics launches with
                                     dist_offset = 0..n-1, then agx_counter_add(dist_counter, n)) replays with fresh draws. */
    uint32_t dist_offset;
    uint32_t dist_pad_;
    const float* target_position; /* [N,3] or NULL (= zeros) */
    /* per-env parameters; NULL = use the AgxHp1Config constant.  Written on reset. */
    float* tau_inc;           /* [N,M] */
    float* tau_dec;           /* [N,M] */
    float* k_thrust;          /* [N,M] */
    float* K_pos;             /* [N,3] */
    float* K_vel;
    float* K_rot;
    float* K_angvel;
    float* bounds_min;        /* [N,3] env bounds (reset); may be NULL = bounds_lo_min / bounds_hi_min */
    float* bounds_max;
    /* derived states (BaseMultirotor.update_states); each may be NULL = not materialised */
    float* euler;             /* [N,3] */
    float* vehicle_orientation; /* [N,4] */
    float* vehicle_linvel;    /* [N,3] */
    float* body_linvel;       /* [N,3] */
    float* body_angvel;       /* [N,3] */
    float* body_wrench;       /* [N,6] net base-frame wrench about the COM of the last physics step, or NULL */
    /* position-task outputs */
    float* obs;               /* [N,13] */
    float* reward;            /* [N] */
    uint8_t* terminations;    /* [N] bool ("crashes") */
    uint8_t* truncations;     /* [N] bool */
    uint8_t* reset_mask;      /* [N] bool, envs reset (or to be reset) this step; may be NULL */
    int32_t* any_reset;       /* [32] device scratch, 16-byte aligned, zero-initialised by the caller once and then always
                                 used with the same num_envs: [0] flag + [1] block-arrival counter (two-launch path);
                                 [2] error word of the chained step's bounded waits (agx_hp1_check);
                                 [4..7] per-step flags, [8..15] four 64-bit arrival counters (single-launch path, hp1.cu) */
    uint32_t* episode_count;  /* [N] device-RNG counter word, incremented per reset */
    float* fresh_vel;         /* [6][N] scratch (SoA): post-physics body lin/ang velocity, written by the fused step
                                 when the stale-observation quirk is on and no derived array is materialised; the
                                 conditional pass then only patches obs[:,7:13] instead of recomputing.  May be NULL. */
    unsigned long long* publish_ctr; /* device u64[4] on a cache line of its own (zero-initialised once) or NULL: the single-launch step
                                        bumps publish_ctr[T & 3] once per tile when the tile's outputs are in memory -- what
                                        agx_obs_gather_push waits on (agx_hp1_task_step_is_chained) */
    uint32_t* tile_sync;      /* [2][ceil(N/32)] device scratch, zero-initialised once: per-tile claim / done counters that
                                 chain consecutive single-launch steps tile by tile (hp1.cu "chained steps").
                                 NULL = the step always takes the two-launch path. */
} AgxHp1Buffers;

/* explicit uniform draws u in [0,1) for agx_hp1_reset, in the reference's call order */
typedef struct AgxHp1ResetDraws {
    const float* bounds_lo;   /* [N,3]  IGE_env_manager.py:513-516 */
    const float* bounds_hi;   /* [N,3]  IGE_env_manager.py:517-519 */
    const float* state;       /* [N,13] base_multirotor.py:182 */
    const float* K_pos;       /* [N,3] each, or NULL when gains are not randomised */
    const float* K_vel;
    const float* K_rot;
    const float* K_angvel;
    const float* tau_inc;     /* [N,M] motor_model.py:141-143 */
    const float* tau_dec;     /* [N,M] motor_model.py:145-147 */
    const float* thrust;      /* [N,M] motor_model.py:148-150 */
    const float* k_thrust;    /* [N,M] motor_model.py:151-154 (NULL unless use_rps) */
} AgxHp1ResetDraws;

struct AgxObsGatherPush;
int agx_abi_version(void);
const char* agx_last_error(void);
/* sizeof() of the ABI structs as compiled into the library (binding self-check):
 * which = 0 AgxHp1Config, 1 AgxHp1Buffers, 2 AgxHp1ResetDraws, 3 AgxHp2Scene, 4 AgxHp2Sensor,
 * 5 AgxNavRewardParams, 6 AgxImuConfig, 7 AgxLidarNavRewardParams, 8 AgxHp2Noise, 9 AgxE2ERewardParams, 10 AgxObsGatherPush */
uint64_t agx_sizeof(int which);

/* Host buffers the kernels can address directly (pinned, portable, mapped: cudaHostAlloc).
 * Any of AgxHp1Buffers' `actions` (read) and `obs` / `reward` / `terminations` / `truncations`
 * (write-only in the fused task step) may point into such a buffer: the step then loads its inputs
 * from and stores its results to host memory over PCIe inside the one launch, without staging
 * copies ("host I/O" mode; the caller synchronises the stream before reading).  The reference moves
 * these tensors with .cpu() / .to("cuda") around task.step (e.g.
 * rl_training/sample_factory/end_to_end_training/enjoy.py:70-91). */
int agx_host_alloc(uint64_t bytes, void** out);
int agx_host_free(void* p);

/* Physics only: `physics_steps` x (update_states -> controller -> allocation -> motor -> drag ->
 * disturbance -> integrate).  Replaces the body of EnvManager.step's loop
 * (env_manager/env_manager.py:426-428 = robots/base_multirotor.py:296-307 + gym.simulate,
 * IGE_env_manager.py:444-449,477,486-495).  Derived-state arrays, when given, receive the
 * PRE-physics values of the last step (the reference's staleness). */
int agx_hp1_physics_step(const AgxHp1Config* cfg, const AgxHp1Buffers* buf, void* stream);

/* Fused PositionSetpointTask.step (task/position_setpoint_task/position_setpoint_task.py:152-182):
 * physics, sim_steps += 1, reward + crash (:245-282), truncation (:172-174), optional in-kernel
 * reset (AGX_F_DEVICE_RNG_RESET), observation (:194-203).  Without AGX_F_DEVICE_RNG_RESET the
 * envs to reset are only flagged (reset_mask, any_reset[0]) and the caller follows with
 * agx_hp1_reset + agx_hp1_refresh. */
int agx_hp1_position_task_step(const AgxHp1Config* cfg, const AgxHp1Buffers* buf, void* stream);
/* The chained step with its observation gather in ONE call (three launches, one host round trip -- at ~10 us per step the host's
 * launch path is the next bottleneck): agx_obs_gather_gate(gate_read_done, gate_need_epoch) on `stream` unless gate_read_done is
 * NULL, agx_hp1_position_task_step(cfg, buf, stream), agx_obs_gather_push(push, push_stream).  See those three. */
int agx_hp1_position_task_step_gathered(const AgxHp1Config* cfg, const AgxHp1Buffers* buf, void* stream, const uint32_t* gate_read_done,
                                        uint32_t gate_need_epoch, uint32_t* gate_error_word, const struct AgxObsGatherPush* push,
                                        void* push_stream);
/* Same call; additionally records the cudaEvent_t `ev_after_main` between the main kernel and the
 * conditional refresh pass, so a caller can time the dominant kernel alone (bench.py roofline). */
int agx_hp1_position_task_step_profiled(const AgxHp1Config* cfg, const AgxHp1Buffers* buf, void* stream,
                                        void* ev_after_main);

/* 1 when agx_hp1_position_task_step(cfg, buf) takes the single-launch path whose consecutive launches are chained per
 * 32-env tile (all CTAs of a step co-resident; device-RNG reset + strict stale observation + tile_sync given), 0 when it takes
 * the two-launch path, negative on error.  Step T (0-based count of such launches since tile_sync / any_reset were zeroed) is
 * complete -- observation included -- when buf->publish_ctr[T & 3] has reached (T / 4 + 1) * ceil(N / 32):
 * that is the (ready_ctr, ready_target) pair agx_obs_gather_push waits on.  (Multi-GPU: the step kernel itself never
 * touches NVLink and never waits for the gather; `obs` is then one slot of a ring of observation buffers the caller rotates and
 * throttles with stream events, see agx_obs_gather_push.) */
int agx_hp1_task_step_is_chained(const AgxHp1Config* cfg, const AgxHp1Buffers* buf);
/* Bound of every in-kernel wait (chained steps, observation gather), wall clock; default 20 s.  On expiry a kernel records an
 * error word and goes on (no trap, the context survives); the next agx_hp1_check / agx_obs_gather_check returns AGX_E_TIMEOUT. */
int agx_set_spin_timeout_ms(uint64_t ms);
/* *counter += n on `stream` (one thread): advances the device-resident draw counter of the in-kernel disturbance. */
int agx_counter_add(uint32_t* counter, uint32_t n, void* stream);
/* Synchronises `stream` and returns AGX_E_TIMEOUT if a wait of the chained step expired since any_reset was zeroed. */
int agx_hp1_check(const AgxHp1Buffers* buf, void* stream);

/* Masked re-initialisation, EnvManager.reset_idx for a robot-only scene
 * (env_manager/env_manager.py:273-301 -> IGE_env_manager.py:513-519, base_multirotor.py:177-205,
 * base_lee_controller.py:101-118, motor_model.py:140-154).  `mask` [N] bool selects envs.
 * draws != NULL: uniforms supplied by the caller (torch RNG, reference order);
 * draws == NULL: device RNG (same stream layout as the fused step). */
int agx_hp1_reset(const AgxHp1Config* cfg, const AgxHp1Buffers* buf, const uint8_t* mask,
                  const AgxHp1ResetDraws* draws, void* stream);

/* BaseMultirotor.update_states for ALL envs (base_multirotor.py:287-294, called at :204-205)
 * plus the position-task observation when buf->obs != NULL.  only_if_flag != 0: the pass is a
 * no-op unless buf->any_reset[0] != 0 (and it clears the flag). */
int agx_hp1_refresh(const AgxHp1Config* cfg, const AgxHp1Buffers* buf, int only_if_flag, void* stream);

/* --------------------------------------------------------------------------------------
 * SURVEY 8(f) rows 3 and 4: NavigationTask epilogue and IMU (small per-env kernels; the
 * random draws are inputs, drawn by the host with torch in the reference's call order)
 * -------------------------------------------------------------------------------------- */
/* reward_parameters of config/task_config/navigation_task_config.py:30-49, in that order:
 * pos_reward_{magnitude,exponent}, very_close_to_goal_reward_{magnitude,exponent},
 * getting_closer_reward_multiplier, {x,z,yawrate}_action_diff_penalty_{magnitude,exponent},
 * {x,z,yawrate}_absolute_action_penalty_{magnitude,exponent}, collision_penalty */
typedef struct AgxNavRewardParams {
    float v[18];
} AgxNavRewardParams;

/* NavigationTask.compute_rewards_and_crashes + compute_reward
 * (task/navigation_task/navigation_task.py:397-418, 436-521).
 *   robot_state [N,stride] (position in columns 0..2), vehicle_orientation [N,4], target_position [N,3],
 *   crashes [N] bool, actions / prev_actions [N,4] (obs_dict robot_actions / robot_prev_actions);
 *   pos_error [N,3]: in = last step's vehicle-frame position error, out = this step's;
 *   pos_error_prev [N,3] out = the value pos_error held on entry; rewards [N] out. */
int agx_nav_reward(int num_envs, const float* robot_state, int robot_state_stride, const float* vehicle_orientation,
                   const float* target_position, const uint8_t* crashes, const float* actions, const float* prev_actions,
                   float curriculum_progress_fraction, const AgxNavRewardParams* params, float* pos_error, float* pos_error_prev,
                   float* rewards, void* stream);

/* NavigationTask.process_obs_for_task (navigation_task.py:369-395), observation columns 0..16 of obs
 * [N,obs_stride]; columns 17.. (the VAE latents) are not touched.  u_vec, u_euler [N,3]: the two
 * torch.rand_like draws of :374 and :382, in that order. */
int agx_nav_obs(int num_envs, const float* robot_state, int robot_state_stride, const float* vehicle_orientation, const float* euler,
                const float* body_linvel, const float* body_angvel, const float* robot_actions, const float* target_position,
                const float* u_vec, const float* u_euler, float* obs, int obs_stride, void* stream);

typedef struct AgxImuConfig {
    int32_t world_frame;     /* BaseImuConfig.world_frame */
    int32_t enable_noise, enable_bias;
    float sqrt_dt;           /* sqrt(sim dt), base_sensor.py:23 */
    float g_world[3];        /* gravity * (1 - gravity_compensation), imu_sensor.py:61-63 */
    float bias_std[6], noise_std[6], max_meas[6]; /* base_imu_config.py:16-43 */
} AgxImuConfig;

/* IMUSensor.update (sensors/imu_sensor.py:85-131).  force [N,force_stride]: the IMU link's force-sensor
 * reading (columns 0..2), robot_state [N,stride] (orientation in columns 3..6), body_angvel [N,3],
 * sensor_quats [N,4]; n_noise, n_bias [N,6]: torch.randn draws of sample_noise (:74-77) and update_bias
 * (:79-83), in that order; bias [N,6] in/out (random walk); imu_meas [N,6] out (accel, gyro). */
int agx_imu_update(int num_envs, const AgxImuConfig* cfg, const float* force, int force_stride, const float* mass,
                   const float* robot_state, int robot_state_stride, const float* body_angvel, const float* sensor_quats,
                   const float* n_noise, const float* n_bias, float* bias, float* imu_meas, void* stream);

/* ---- LiDARNavigationTask epilogue (task/lidar_navigation_task/lidar_navigation_task.py) ---------------- */

/* LiDARNavigationTask.process_image_observation up to the min-pooling (:313-347): for every return of the
 * world-frame point cloud  range = |p - robot_position|  (> max_range or < min_range -> invalid_value, :320-321),
 * the per-pixel time to collision along the robot's world velocity (:327-335), then
 *   image_ds [N, height/pool_h, width/pool_w] = min-pool (pool_h x pool_w, stride = window; -max_pool2d(-x), :346-347)
 *   time_to_collision [N] = clamp(min over ALL pixels, 0, ttc_max)  (:339; ttc_max is also the value of a pixel
 *   the robot is not moving towards).
 * pointcloud [N,height,width,3] (depth_range_pixels with the sensor dimension squeezed); robot_state [N,stride] with
 * the position in columns 0..2 and the world linear velocity in columns 7..9.  The task's own noise model (:286-310,
 * torch RNG) and the final 1/x (:351) stay with the caller.  The reference hard-codes max_range = invalid_value =
 * ttc_max = 10, min_range = 0.2, pool 3 x 6 on a 48 x 120 image. */
int agx_lidar_nav_pool(int num_envs, int height, int width, int pool_h, int pool_w, const float* pointcloud,
                       const float* robot_state, int robot_state_stride, float max_range, float min_range,
                       float invalid_value, float ttc_max, float* image_ds, float* time_to_collision, void* stream);

/* reward_parameters of LiDARNavigationTask in the order of config/task_config/lidar_navigation_task_config.py:28-51:
 * pos_reward_{magnitude,exponent}, very_close_to_goal_reward_{magnitude,exponent},
 * vel_direction_component_reward_magnitude, {x,y,z,yawrate}_action_diff_penalty_{magnitude,exponent},
 * {x,y,z,yawrate}_absolute_action_penalty_{magnitude,exponent}, collision_penalty */
typedef struct AgxLidarNavRewardParams {
    float v[22];
    int32_t radar_variant; /* 0: LiDARNavigationTask.  1: RadarNavigationTask (task/radar_navigation_task/radar_navigation_task.py), whose
                              compute_reward differs in one term: the x-velocity penalty is taken on clamp(vx, max=0) instead of
                              clamp(vx, min=0) (:251 there vs lidar_navigation_task.py:619) */
} AgxLidarNavRewardParams;

/* LiDARNavigationTask.compute_rewards_and_crashes + compute_reward (:471-499, :554-720).
 *   robot_state [N,stride] (position in columns 0..2), vehicle_orientation [N,4], target_position [N,3],
 *   euler [N,3] (robot_euler_angles), target_yaw [N], vehicle_linvel / body_angvel [N,3], crashes [N] bool,
 *   actions / prev_actions [N,4] (the task's current_action / prev_action), time_to_collision [N] (last value
 *   written by agx_lidar_nav_pool);
 *   pos_error [N,3] in = last step's vehicle-frame position error, out = this step's; pos_error_prev [N,3] out =
 *   the value pos_error held on entry; rewards [N] out. */
int agx_lidar_nav_reward(int num_envs, const float* robot_state, int robot_state_stride, const float* vehicle_orientation,
                         const float* target_position, const float* euler, const float* target_yaw, const float* vehicle_linvel,
                         const float* body_angvel, const uint8_t* crashes, const float* actions, const float* prev_actions,
                         const float* time_to_collision, float curriculum_progress_fraction, const AgxLidarNavRewardParams* params,
                         float* pos_error, float* pos_error_prev, float* rewards, void* stream);

/* LiDARNavigationTask.process_obs_for_task (:440-469): observation columns 0..16 of obs [N,obs_stride], then columns
 * 17..17+num_lidar-1 = lidar_obs [N,num_lidar] (downsampled_lidar_data; NULL or num_lidar = 0: untouched).
 * u_vec, u_euler [N,3]: the two torch.rand_like draws of :446 and :456, in that order. */
int agx_lidar_nav_obs(int num_envs, const float* robot_state, int robot_state_stride, const float* vehicle_orientation,
                      const float* euler, const float* body_linvel, const float* body_angvel, const float* robot_actions,
                      const float* target_position, const float* target_yaw, const float* u_vec, const float* u_euler,
                      const float* lidar_obs, int num_lidar, float* obs, int obs_stride, void* stream);


/* ---- motor-command ("end to end") position tasks: position_setpoint_task_sim2real_end_to_end / _px4 ------ */

/* the constants in which the two tasks' compute_reward differ
 * (task/position_setpoint_task_sim2real_end_to_end/...py:267-311 | task/position_setpoint_task_sim2real_px4/...py:268-312) */
typedef struct AgxE2ERewardParams {
    float z_error_scale;                 /* 11 | 13        (:283) */
    float upright_gain2, upright_exp2;   /* 0, 0 | 2.5, 2  (:288) */
    float align_gain1, align_exp1;       /* 6, 5 | 4, 5    (:292) */
    float align_gain2, align_exp2;       /* 0, 0 | 2, 2 */
    float angvel_gain;                   /* 0.3 | 0.75     (:294) */
    float hover_thrust;                  /* 9.81 * 0.372 / 4 | 9.81 * 1.6559999883174896 / 4   (:297) */
    float towards_gain_pos, towards_gain_neg; /* 10, 15 | 50, 100 (:301) */
    float action_diff_gain;              /* 1.3 | 0.5      (:304) */
    float crash_dist;                    /* task_config.crash_dist */
} AgxE2ERewardParams;

/* compute_rewards_and_crashes + compute_reward.  robot_state [N,stride] (position 0..2, orientation xyzw 3..6, WORLD linear velocity
 * 7..9), body_angvel [N,3] (robot_body_angvel, stale like the reference's), target_position [N,3] or NULL (= 0), actions /
 * prev_actions [N,4] (motor commands after process_actions_for_task), prev_pos_error [N,3]; crashes [N] bool: OR-ed with
 * |pos error| > crash_dist; rewards [N] out. */
int agx_e2e_reward(int num_envs, const float* robot_state, int robot_state_stride, const float* body_angvel, const float* target_position,
                   const float* actions, const float* prev_actions, const float* prev_pos_error, const AgxE2ERewardParams* params,
                   uint8_t* crashes, float* rewards, void* stream);

/* process_obs_for_task (:204-229): obs[:, 0:15] = noisy position error (3), rotation-6D of the noisy ZYX Euler angles (6), noisy WORLD
 * linear velocity (3), noisy body rates (3).  noise [N,12]: the four torch.normal draws in the method's order, side by side. */
int agx_e2e_obs(int num_envs, const float* robot_state, int robot_state_stride, const float* body_angvel, const float* target_position,
                const float* noise, float* obs, int obs_stride, void* stream);

/* ---- setpoint-command sim2real position tasks: position_setpoint_task_sim2real / _acceleration_sim2real (lmf2) ---- */

/* compute_rewards_and_crashes + compute_reward (task/position_setpoint_task_sim2real/...py:230-339, variant 0;
 * task/position_setpoint_task_acceleration_sim2real/...py:239-356, variant 1).  robot_state [N,stride] (position 0..2, orientation
 * 3..6), vehicle_orientation [N,4], body_linvel [N,3] (both stale like the reference's), target_position [N,3] or NULL, prev_dist [N]
 * (distance to the target before the step), actions / prev_actions [N,4]: variant 0 = the task's actions / prev_actions; variant 1 =
 * the actions (rotated in the kernel by vehicle_orientation -> actions_vehicle_frame [N,4] out, may be NULL) /
 * prev_actions_vehicle_frame.  crashes [N] bool in/out (|= distance > 10), rewards [N] out (-50 where crashed). */
int agx_s2r_reward(int num_envs, int variant, const float* robot_state, int robot_state_stride, const float* vehicle_orientation,
                   const float* body_linvel, const float* target_position, const float* prev_dist, const float* actions,
                   const float* prev_actions, float* actions_vehicle_frame, uint8_t* crashes, float* rewards, void* stream);

/* process_obs_for_task (:202-228): obs[:, 0:17] = noisy position error, quaternion of the noisy Euler angles, noisy body velocities,
 * robot_actions.  noise [N,12]: the four torch.randn_like draws (euler, position, body linvel, body angvel) side by side, unscaled.
 * robot_state's orientation is multiplied by sign(qw) IN PLACE, as the reference does (:204-207). */
int agx_s2r_obs(int num_envs, float* robot_state, int robot_state_stride, const float* body_linvel, const float* body_angvel,
                const float* robot_actions, const float* target_position, const float* noise, float* obs, int obs_stride, void* stream);

/* ---- random wrench disturbance, device RNG -------------------------------------------------------------- */

/* BaseMultirotor.apply_disturbance (robots/base_multirotor.py:213-234) as one launch: disturbance [N,6] (device) = with probability
 * prob a body-0 force ~ U(-max, max)^3 and torque ~ U(-max, max)^3, else zero; feeds AgxHp1Buffers.disturbance.
 * max_force_and_torque: HOST array of six floats (cfg.disturbance.max_force_and_torque_disturbance).  Device RNG (Philox4x32-10,
 * counter = (env_id_offset + env, counter, block, 'DIST'), key = seed): same distributions as the reference's torch.bernoulli +
 * 2 x rand_like, its own stream, independent of sharding; `counter` advances once per physics step. */
int agx_disturbance_draw(int num_envs, int env_id_offset, float prob, const float* max_force_and_torque, uint64_t seed,
                         uint32_t counter, float* disturbance, void* stream);

/* ---- dynamic obstacles ("dynamic_env": env_manager/obstacle_manager.py:40-44 + PhysX) ------------------- */

/* Kinematic advance of every obstacle by `substeps` physics steps of `dt`.  asset_state [N,A,asset_stride] rows
 * x y z qx qy qz qw vx vy vz wx wy wz (env_asset_state_tensor, IGE_env_manager.py:315-317), in/out; twist [N,A,6] =
 * env_actions (linear, angular velocity, world frame; written into the state before EVERY physics step like
 * ObstacleManager.pre_physics_step does) or NULL = keep the velocities the state holds.  Per physics step (our spec -- PhysX
 * is not observable; the robot integrator's form): v *= max(0, 1 - dt linear_damping), w likewise, x += dt v,
 * q = normalize(dq(w dt) (x) q).  The caller re-poses the ray-cast scene afterwards (agx_hp2_update_scene). */
int agx_obstacle_step(int num_envs, int num_assets, float* asset_state, int asset_stride, const float* twist, float dt, int substeps,
                      float linear_damping, float angular_damping, void* stream);

/* ======================================================================================
 * HP2 -- depth / segmentation / LiDAR ray-caster
 * ====================================================================================== */
#define AGX_HAVE_HP2 1
#define AGX_HP2_MAX_OBJECTS 2048      /* objects (triangle clusters) per env */
#define AGX_NO_HIT_RAY_VAL 1000.0f    /* sensors/warp/warp_kernels/warp_camera_kernels.py:3 */
#define AGX_NO_HIT_SEG_VAL (-2)       /* warp_camera_kernels.py:4 */

/* Per-env triangle scene + BVH.  Replaces WarpEnv (env_manager/warp_env_manager.py:97-189):
 * one wp.Mesh per env built from the concatenated asset meshes, vertices re-transformed by the
 * asset root poses and the BVH refit on reset (:40-54).
 * Geometry is instanced: every object of every env references a TEMPLATE (a triangle list in the
 * object frame, <= tris_per_object triangles; larger meshes are split into several templates
 * by the host) and carries a pose.  agx_hp2_update_scene writes the world-space triangles and
 * builds the per-env BVH (Morton-sorted implicit balanced binary tree over objects). */
typedef struct AgxHp2Scene {
    int32_t num_envs;
    int32_t num_objects;        /* K objects per env (same for all envs), 1..AGX_HP2_MAX_OBJECTS */
    int32_t leaves_pow2;        /* P = smallest power of two >= K */
    int32_t tris_per_object;    /* L triangle slots per object (padded with degenerate triangles) */
    int32_t num_templates;
    int32_t obj_pose_stride;    /* floats between consecutive object poses (13 for env_asset_state_tensor rows) */
    const int32_t* tmpl_tri_offset; /* [T+1] first triangle of each template */
    const float* tmpl_tris;     /* [Ft,9] object-frame v0,v1,v2 */
    const int32_t* tmpl_seg_base; /* [Ft] asset_vertex_segmentation_value of the face's first vertex (assets/warp_asset.py:113) */
    const int32_t* tmpl_seg_mask; /* [Ft] variable_segmentation_mask (assets/warp_asset.py:114-116) */
    const float* obj_pose;      /* [E,K,stride] x y z qx qy qz qw ... (env_asset_state_tensor, IGE_env_manager.py:315-317) */
    const int32_t* obj_template;    /* [E,K] */
    const int32_t* obj_seg_counter; /* [E,K] segmentation counter of the instance (warp_env_manager.py:76-80) */
    const float* bounds_min;    /* [E,3] env bounds used to normalise Morton codes, or NULL */
    const float* bounds_max;
    /* device storage owned by the caller, layout defined by the library: */
    float* tris;                /* [E][K*L][12]  (v0.xyz, seg bits | e1.xyz, 0 | e2.xyz, 0) */
    float* nodes;               /* [E][2P-1][8]  (lo.xyz, 0 | hi.xyz, 0), heap order, leaves last */
    int32_t* leaf_object;       /* [E][max(P,4)] object index of each Morton-sorted leaf, -1 = empty */
    int32_t* face_offset;       /* [E][K] index of each object's first triangle in the env's concatenated mesh
                                   (the face id of the normal+faceID sensors); may be NULL if those are unused */
    /* optional culling aid: templates that are boxes carry their object-frame oriented box; leaves whose
     * (padded) world OBB the ray misses skip their 12 triangle tests.  Culling only -- results unchanged. */
    const float* tmpl_obb;      /* [T][16] centre.xyz, axis0.xyz, axis1.xyz, axis2.xyz, half.xyz, valid(0/1); or NULL */
    float* obb;                 /* [E][K][16] world-frame boxes written by agx_hp2_update_scene; NULL iff tmpl_obb is NULL */
} AgxHp2Scene;

#define AGX_SENSOR_CAMERA 0              /* warp_camera_kernels.py:125-282 */
#define AGX_SENSOR_LIDAR 1               /* warp_lidar_kernels.py:13-86,130-194 */
#define AGX_SENSOR_STEREO_CAMERA 2       /* warp_stereo_camera_kernels.py (depth/range +- seg with occlusion re-cast) */
#define AGX_SENSOR_NORMAL_FACEID_CAMERA 3 /* warp_camera_kernels.py:70-121 */
#define AGX_SENSOR_NORMAL_FACEID_LIDAR 4  /* warp_lidar_kernels.py:90-126 */

/* One sensor type on every robot.  Replaces WarpSensor.update (sensors/warp/warp_sensor.py:177-200)
 * = pose compose (:180-187) + WarpCam/WarpLidar.capture (warp_cam.py:172-182, warp_lidar.py) +
 * apply_range_limits (:202-220) + normalize_observation (:222-225). */
typedef struct AgxHp2Sensor {
    int32_t kind;               /* AGX_SENSOR_* */
    int32_t width, height, num_sensors;
    int32_t calculate_depth;    /* camera: depth image (1) or range image (0) */
    int32_t return_pointcloud, pointcloud_in_world_frame, segmentation;
    int32_t fuse_epilogue;      /* apply range limits + normalisation in the kernel (noise disabled) */
    int32_t normalize_range;
    int32_t c_x, c_y;           /* warp_cam.py:63-64 */
    float kinv[9];              /* upper-left 3x3 of K^-1 (warp_cam.py:43-62) */
    float far_plane;            /* = max_range (warp_cam.py:21) */
    float max_range, min_range, far_out_of_range_value, near_out_of_range_value;
    float frame_quat[4];        /* sensor data frame (warp_sensor.py:100-105) */
    float baseline;             /* stereo baseline (stereo_camera_config.py:9) */
    int32_t normal_in_world_frame; /* normal+faceID sensors */
    int32_t robot_pose_stride;  /* floats between robot poses (13 for robot_state_tensor rows) */
    int32_t pad_;
    const float* robot_pose;    /* [E,stride] x y z qx qy qz qw ... */
    const float* mount;         /* [E,S,7] sensor_local_position + sensor_local_orientation */
    const float* ray_table;     /* [H,W,3] LiDAR ray vectors (warp_lidar.py:40-64) or NULL */
    float* pixels;              /* [E,S,H,W], or [E,S,H,W,3] for pointclouds / normals (depth_range_pixels) */
    int32_t* seg_pixels;        /* [E,S,H,W] segmentation ids (or face ids for the normal+faceID kinds), or NULL */
} AgxHp2Sensor;

/* bytes the caller must allocate for scene->tris / nodes / leaf_object (per env) */
uint64_t agx_hp2_scene_bytes(int num_objects, int tris_per_object, int which /*0 tris, 1 nodes, 2 leaf_object, 3 face_offset, 4 obb*/);

/* Re-transform triangles + rebuild the BVH of the envs selected by `mask` ([E] bool, NULL = all).
 * Replaces WarpEnv.reset_idx (warp_env_manager.py:40-54). */
int agx_hp2_update_scene(const AgxHp2Scene* scene, const uint8_t* mask, void* stream);

/* Cast every ray of every sensor of every env.  Replaces WarpSensor.update. */
int agx_hp2_cast(const AgxHp2Scene* scene, const AgxHp2Sensor* sensor, void* stream);

/* Collision flag (SURVEY 8a row a14).  Replaces EnvManager.compute_observations
 * (env_manager/env_manager.py:358-362: crashes += |PhysX contact force on body 0| > threshold).
 * PhysX contacts are not reproducible; the flag is geometric: the robot's collision sphere
 * (centre = robot position, `radius`) overlaps the env's triangle mesh.
 *   crashes  [E] bool : OR-ed with the overlap flag (the reference accumulates with +=)
 *   min_dist [E] f32  : distance from the sphere centre to the closest triangle, or NULL */
int agx_hp2_collide(const AgxHp2Scene* scene, const float* robot_pose, int robot_pose_stride, float radius,
                    uint8_t* crashes, float* min_dist, void* stream);


/* ======================================================================================
 * Multi-GPU: observation all-gather over NVLink peer memory (SURVEY section 8e)
 * ====================================================================================== */
#define AGX_MAX_PEERS 16

/* One-shot all-gather written as ONE kernel of P2P stores (no NCCL on the step path): every rank
 * copies its `bytes` (multiple of 16) of `local` into slot `rank` of EVERY peer's gathered buffer
 * (peer_bufs[p] + rank*bytes, pointers obtained from a symmetric-memory rendezvous), publishes
 * `epoch` into each peer's flag word `peer_flags[p][rank]` with system-scope release semantics, and
 * the kernel does not retire before the flags of all peers show `epoch` for this rank -- so work
 * queued behind it on the stream sees the complete [world*bytes] buffer.  The reference has no
 * distributed code; this replaces what would be torch.distributed.all_gather_into_tensor.
 *   peer_bufs / peer_flags : DEVICE arrays of `world` device pointers
 *   scratch                : device uint32 (zero-initialised once), block-arrival counter
 *   epoch                  : strictly increasing per call, starting at 1 */
int agx_p2p_allgather(const void* local, void* const* peer_bufs, uint32_t* const* peer_flags, int world, int rank,
                      uint64_t bytes, uint32_t epoch, uint32_t* scratch, void* stream);

/* ---- pipelined observation all-gather (SURVEY 8e: the one collective of the step path) ---------------------------------
 * Split form of agx_p2p_allgather for use BESIDE the chained steps: the PUSH (sender side) runs on a side stream with a few
 * CTAs while the next steps compute, the WAIT (receiver side) runs on the consumer's stream just before the gathered buffer is
 * read.  Neither is on the step kernel's critical path.
 *
 * agx_obs_gather_push: optionally wait until *ready_ctr >= ready_target (the step that produces `local` has published it: see
 * agx_hp1_task_step_is_chained; NULL = `local` is already complete in stream order) -- a ONE-WARP gate kernel does the waiting and the
 * push kernel is its programmatic dependent, so no push CTA is resident while it would only wait --, copy the `bytes` (multiple of 16) of `local`
 * into slot `rank` of every rank's gathered buffer (peer_bufs[p] + rank * bytes; the own slot is skipped when `local` already is
 * that slot), then -- when all stores of this rank have been performed at system scope -- publish `epoch` into flag word
 * peer_flags[p][flag_slot * AGX_MAX_PEERS + rank] on every rank p.  The kernel never waits for a peer.  Pushes into different ring
 * slots may run concurrently (one stream and one scratch block per slot); re-use of a slot is ordered by the caller
 * (agx_obs_gather_gate on `read_done`, or plain stream order).
 *   peer_bufs / peer_flags : DEVICE arrays of `world` device pointers (symmetric-memory rendezvous)
 *   scratch                : device uint32[4] of this ring slot, zero-initialised once
 *   error_word             : device uint32, zero-initialised once (agx_obs_gather_check)
 *   epoch                  : strictly increasing per push, starting at 1
 *   max_ctas               : upper bound of the grid (0 = default 24): the pushes share the GPU with the chained step */
typedef struct AgxObsGatherPush {
    const void* local;
    void* const* peer_bufs;
    uint32_t* const* peer_flags;
    int32_t world, rank;
    uint64_t bytes;
    uint32_t epoch;
    int32_t max_ctas;
    const unsigned long long* ready_ctr;
    uint64_t ready_target;
    uint32_t* scratch;
    uint32_t* error_word;
    int32_t flag_slot;
    int32_t pad_;
    uint32_t* read_done;   /* device uint32 of this ring slot or NULL: receives `epoch` (release, gpu scope) as soon as every CTA has
                              finished READING `local` -- before the NVLink drain; agx_obs_gather_gate waits on it */
    void* mc_buf;          /* NVSwitch multicast address of the SAME gathered buffer (symmetric-memory multicast_ptr) or NULL.  When set,
                              every 16 bytes leave this GPU ONCE (`multimem.st`) and the switch replicates them into all ranks' buffers:
                              the push's store count and NVLink egress no longer grow with the world size (7x at 8 GPUs).  The flag
                              words are still written peer by peer. */
} AgxObsGatherPush;
int agx_obs_gather_push(const AgxObsGatherPush* a, void* stream);
/* Ring-slot gate for a producer that runs ahead of its pushes: a one-warp kernel, launched with programmatic stream serialization
 * on the producer's stream, that lets the launch behind it start only once *read_done >= need_epoch (wrap-safe), i.e. once the push
 * that last read the ring slot the next step is about to overwrite has finished reading it.  Between two chained
 * agx_hp1_position_task_step launches it keeps their per-tile chaining (no event, no stream-level wait). */
int agx_obs_gather_gate(const uint32_t* read_done, uint32_t need_epoch, uint32_t* error_word, void* stream);
/* Receiver side: one tiny kernel that retires when my_flags[flag_slot * AGX_MAX_PEERS + q] >= epoch for every rank q < world
 * (wrap-safe compare), i.e. when every rank's rows of `epoch` have landed in this rank's gathered buffer of that ring slot; work
 * queued behind it on `stream` may read it. */
int agx_obs_gather_wait(const uint32_t* my_flags, int flag_slot, int world, uint32_t epoch, uint32_t* error_word, void* stream);
/* Synchronises `stream`; AGX_E_TIMEOUT if a push / wait gave up (bounded by agx_set_spin_timeout_ms). */
int agx_obs_gather_check(const uint32_t* error_word, void* stream);
int agx_obs_gather_set_timeout_ns(uint64_t ns);

/* Sensor noise + range limits + normalisation, one pass, device RNG.  Replaces WarpSensor.apply_noise +
 * apply_range_limits + normalize_observation (sensors/warp/warp_sensor.py:202-247) when the sensor's noise model is enabled
 * (agx_hp2_cast then runs with fuse_epilogue = 0 and leaves raw ranges).  Same distributions as the reference --
 * value ~ N(p - mean_offset, std_a p^2 + std_b p + std_c), dropout with probability pixel_dropout_prob -> near value, then
 * > max_range -> far value, < min_range -> near value (on the norm of a sensor-frame point), / max_range -- but its own stream:
 * Philox4x32-10, counter (pixel lo, pixel hi, frame, component), key = seed.  The torch-RNG path with the reference's draw
 * order is the host's (aerial_gym_simulator_b200/sensors/noise.py). */
typedef struct AgxHp2Noise {
    int32_t components;        /* floats per pixel: 1 (depth / range image) or 3 (point cloud) */
    int32_t enable_noise;      /* sensor_noise.enable_sensor_noise */
    int32_t apply_limits;      /* 1 for camera / lidar / stereo images and sensor-frame point clouds (:198-215) */
    int32_t normalize;         /* normalize_range and not pointcloud_in_world_frame (:222-225) */
    float std_a, std_b, std_c, mean_offset, pixel_dropout_prob;   /* cfg.sensor_noise */
    float max_range, min_range, far_out_of_range_value, near_out_of_range_value;
} AgxHp2Noise;

/* pixels: num_pixels * components floats, in place.  first_pixel: GLOBAL index of pixels[0] (env_id_offset x pixels per env on a
 * sharded run, so the noise does not depend on how the envs are split over GPUs).  frame: a counter the caller advances once
 * per render. */
int agx_hp2_noise_limits(float* pixels, uint64_t num_pixels, uint64_t first_pixel, const AgxHp2Noise* cfg, uint64_t seed, uint32_t frame,
                         void* stream);

#ifdef __cplusplus
}
#endif
#endif /* AERIAL_GYM_B200_H_ */
