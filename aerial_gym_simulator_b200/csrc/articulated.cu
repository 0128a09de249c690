// Articulated multirotors: the physics-only step of agx_hp1_physics_step for a robot whose URDF tree has revolute joints
// (DESIGN.md "Articulated robots").  The per-env arithmetic is articulated_core.cuh; this unit holds the kernel and the entry point
// (articulated_prismatic.cu those of robots with prismatic joints; articulated_launch.cuh what the two share).
//
// Layout: one env per thread, every per-body array of the ABA in the thread's own local memory.  The sweeps over the tree index
// those arrays with the run-time parent table, so they cannot live in registers; a warp's 32 envs walk the same tree in lockstep,
// so their accesses coalesce (local memory is interleaved per thread) and stay in L1 / L2.  The alternative -- one warp per env,
// lanes over the bodies of a tree level -- would keep the scratch in registers and shuffles but leave most lanes idle on a
// 9-body tree whose levels are 1, 4 and 4 bodies wide, and the controller / motor part of the sub-step (a third of its
// instructions) would run on one lane.  DESIGN.md records the measured cost.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/aerial_gym_b200.h"
#include "agx_common.cuh"
#include "articulated_core.cuh"
#include "articulated_launch.cuh"

using namespace agx;

namespace {

template <int M, int NB>
__global__ void __launch_bounds__(kArtThreads)
articulated_step_kernel(const __grid_constant__ AgxHp1Config cfg, const __grid_constant__ AgxHp1Buffers buf,
                        const __grid_constant__ AgxArticulation art) {
    const int env = blockIdx.x * blockDim.x + threadIdx.x;
    if (env >= cfg.num_envs) return;
    art_env_step<M, NB>(cfg, buf, art, env);
}

// ---- the step with the IMU input of one body (agx_hp1_articulated_step_imu): articulated_step_kernel plus one [9] store per env
template <int M, int NB>
__global__ void __launch_bounds__(kArtThreads)
articulated_step_imu_kernel(const __grid_constant__ AgxHp1Config cfg, const __grid_constant__ AgxHp1Buffers buf,
                            const __grid_constant__ AgxArticulation art, int imu_body, float* __restrict__ imu_input) {
    const int env = blockIdx.x * blockDim.x + threadIdx.x;
    if (env >= cfg.num_envs) return;
    art_env_step<M, NB, true>(cfg, buf, art, env, imu_body, imu_input);
}

// ---- the step with effort-mode joints (agx_hp1_articulated_step_effort): one [D] read of the commanded torques per env and launch,
// with or without the IMU input
template <int M, int NB, bool IMU>
__global__ void __launch_bounds__(kArtThreads)
articulated_step_effort_kernel(const __grid_constant__ AgxHp1Config cfg, const __grid_constant__ AgxHp1Buffers buf,
                               const __grid_constant__ AgxArticulation art, const __grid_constant__ AgxJointEffort eff, int imu_body,
                               float* __restrict__ imu_input) {
    const int env = blockIdx.x * blockDim.x + threadIdx.x;
    if (env >= cfg.num_envs) return;
    art_env_step<M, NB, IMU, true>(cfg, buf, art, env, imu_body, imu_input, &eff);
}

// ---- the step with the joint forces (agx_hp1_articulated_step_joint_force): the effort kernel's arithmetic plus the rows of
// joint_wrench [N,B,6] and dof_force [N,D] on the last sub-step.  The IMU input and the effort DOFs are resolved at run time (a NULL
// imu_input, an effort table without effort DOFs), so four instantiations cover every robot.  Written straight from the lanes, a
// warp's rows would sit (6 B + D) floats apart and no store would coalesce; instead each lane's art_dynamics writes its env's rows
// into shared memory (6 B + D floats, plus one when that is even, so that the 32 lanes' accesses at the same offset fall in 32
// different banks), and the warp then copies its contiguous spans of joint_wrench and dof_force out with 16-byte stores, as
// articulated_body_state_kernel does.
template <int M, int NB>
__global__ void __launch_bounds__(kArtThreads)
articulated_step_joint_force_kernel(const __grid_constant__ AgxHp1Config cfg, const __grid_constant__ AgxHp1Buffers buf,
                                    const __grid_constant__ AgxArticulation art, const __grid_constant__ AgxJointEffort eff,
                                    int imu_body, float* __restrict__ imu_input, float* __restrict__ joint_wrench,
                                    float* __restrict__ dof_force) {
    extern __shared__ float s_joint_rows[];
    const int lane = threadIdx.x % kWarp;
    const int env0 = blockIdx.x * blockDim.x + threadIdx.x - lane;
    if (env0 >= cfg.num_envs) return;  // whole warps only: the rest of the warp copies below
    const int B = art.num_bodies, D = art.num_dofs, W = 6 * B, st = joint_force_row_stride(B);
    float* s_warp = s_joint_rows + (threadIdx.x - lane) * st;
    const int env = env0 + lane;
    if (env < cfg.num_envs)
        art_env_step<M, NB, true, true, true>(cfg, buf, art, env, imu_body, imu_input, &eff, s_warp + lane * st, s_warp + lane * st + W);
    __syncwarp();
    const int n = min(kWarp, cfg.num_envs - env0);
    copy_warp_rows(joint_wrench + (size_t)env0 * W, s_warp, st, 0, W, n, lane);  // 16-byte aligned: env0 W is a multiple of 32 x 6
    if (D) copy_warp_rows(dof_force + (size_t)env0 * D, s_warp, st, W, D, n, lane);
}

// ---- per-body state (agx_hp1_articulated_body_state) ----------------------------------------------------------------------
// One env per lane, one warp per block.  Each lane builds its env's B rows (13 B floats) in shared memory with art_body_states, the
// rows of the parents serving as the sweep's scratch, so nothing goes to local memory.  Written straight from the lanes, the rows
// of a warp would sit 52 B apart per lane and no store would coalesce; instead the warp copies its contiguous span of body_state
// (32 x 13 B floats) out of shared memory with 16-byte stores.  A lane's row in shared memory is 13 B floats, plus one when 13 B is
// even, so that the 32 lanes' accesses at the same offset fall in 32 different banks.
template <int NB>
__global__ void __launch_bounds__(kBodyThreads)
articulated_body_state_kernel(const __grid_constant__ AgxArticulation art, int num_envs, const float* __restrict__ root_state,
                              int root_stride, float* __restrict__ body_state) {
    extern __shared__ float4 s_body_rows4[];
    float* s_rows = reinterpret_cast<float*>(s_body_rows4);
    const int B = art.num_bodies, D = art.num_dofs;
    const int len = 13 * B, pad = (len & 1) ^ 1;  // floats of one env's rows; the padding that makes the lane stride odd
    const int lane = threadIdx.x;
    const int env0 = blockIdx.x * kBodyThreads;
    const int env = env0 + lane;
    if (env < num_envs)
        art_body_states<NB>(art, root_state + (size_t)env * root_stride, art.dof_state + (size_t)env * 2 * D, s_rows + lane * (len + pad));
    __syncwarp();
    const int total = min(kBodyThreads, num_envs - env0) * len;  // floats of the warp's span
    float* out = body_state + (size_t)env0 * len;               // 16-byte aligned: env0 * len is a multiple of 32 * 13
    const int n4 = total >> 2;
    if (pad == 0) {
        for (int k = lane; k < n4; k += kBodyThreads) reinterpret_cast<float4*>(out)[k] = s_body_rows4[k];
    } else {
        for (int k = lane; k < n4; k += kBodyThreads) {
            const int g = 4 * k, l0 = g / len;
            float v[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int gj = g + j;
                v[j] = s_rows[gj + l0 + (gj - l0 * len >= len ? 1 : 0)];  // + (env of float gj) x pad, pad = 1
            }
            reinterpret_cast<float4*>(out)[k] = make_float4(v[0], v[1], v[2], v[3]);
        }
    }
    for (int g = 4 * n4 + lane; g < total; g += kBodyThreads) out[g] = s_rows[g + (g / len) * pad];
}

}  // namespace

extern "C" int agx_hp1_articulated_body_state(const AgxArticulation* art, int num_envs, const float* root_state, int root_state_stride,
                                              float* body_state, void* stream) {
    int rc = validate_body_state(art, num_envs, root_state, root_state_stride, body_state);
    if (rc) return rc;
    if (num_envs == 0) return AGX_OK;
    const int g = (num_envs + kBodyThreads - 1) / kBodyThreads;
    const int len = 13 * art->num_bodies;
    const size_t smem = sizeof(float) * kBodyThreads * (len + ((len & 1) ^ 1));  // <= 26.75 KB at 16 bodies
    // the kernel has no motors: only the tree size of the instantiation applies
    const auto kern = art_instantiation(4, art->num_bodies, [](auto, auto nb) { return articulated_body_state_kernel<nb>; });
    kern<<<g, kBodyThreads, smem, (cudaStream_t)stream>>>(*art, num_envs, root_state, root_state_stride, body_state);
    return agx_check_launch("articulated_body_state_kernel");
}

extern "C" int agx_hp1_articulated_step(const AgxHp1Config* cfg, const AgxHp1Buffers* buf, const AgxArticulation* art, void* stream) {
    int rc = validate_step(cfg, buf, art, nullptr, false, 0);
    if (rc) return rc;
    if (cfg->num_envs == 0) return AGX_OK;
    const auto kern = art_instantiation(cfg->num_motors, art->num_bodies, [](auto m, auto nb) { return articulated_step_kernel<m, nb>; });
    kern<<<art_blocks(cfg), kArtThreads, 0, (cudaStream_t)stream>>>(*cfg, *buf, *art);
    return agx_check_launch("articulated_step_kernel");
}

extern "C" int agx_hp1_articulated_step_imu(const AgxHp1Config* cfg, const AgxHp1Buffers* buf, const AgxArticulation* art, int imu_body,
                                            float* imu_input, void* stream) {
    int rc = validate_step(cfg, buf, art, nullptr, true, imu_body);
    if (rc) return rc;
    if (!imu_input) return agx_set_error(AGX_E_NULL, "imu_input is NULL");
    if (cfg->num_envs == 0) return AGX_OK;
    const auto kern =
        art_instantiation(cfg->num_motors, art->num_bodies, [](auto m, auto nb) { return articulated_step_imu_kernel<m, nb>; });
    kern<<<art_blocks(cfg), kArtThreads, 0, (cudaStream_t)stream>>>(*cfg, *buf, *art, imu_body, imu_input);
    return agx_check_launch("articulated_step_imu_kernel");
}

extern "C" int agx_hp1_articulated_step_effort(const AgxHp1Config* cfg, const AgxHp1Buffers* buf, const AgxArticulation* art,
                                               const AgxJointEffort* effort, int imu_body, float* imu_input, void* stream) {
    int rc = validate_step(cfg, buf, art, effort, imu_input != nullptr, imu_body);
    if (rc) return rc;
    if (!effort) return agx_set_error(AGX_E_NULL, "effort is NULL");
    if (cfg->num_envs == 0) return AGX_OK;
    const auto kern = art_instantiation(cfg->num_motors, art->num_bodies, [&](auto m, auto nb) {
        return imu_input ? articulated_step_effort_kernel<m, nb, true> : articulated_step_effort_kernel<m, nb, false>;
    });
    kern<<<art_blocks(cfg), kArtThreads, 0, (cudaStream_t)stream>>>(*cfg, *buf, *art, *effort, imu_body, imu_input);
    return agx_check_launch("articulated_step_effort_kernel");
}

extern "C" int agx_hp1_articulated_step_joint_force(const AgxHp1Config* cfg, const AgxHp1Buffers* buf, const AgxArticulation* art,
                                                    const AgxJointEffort* effort, int imu_body, float* imu_input, float* joint_wrench,
                                                    float* dof_force, void* stream) {
    int rc = validate_step(cfg, buf, art, effort, imu_input != nullptr, imu_body);
    if (rc) return rc;
    if (cfg->num_envs == 0) return AGX_OK;
    if (!joint_wrench || (art->num_dofs > 0 && !dof_force)) return agx_set_error(AGX_E_NULL, "joint_wrench/dof_force is NULL");
    if (((uintptr_t)joint_wrench | (uintptr_t)dof_force) & 15)
        return agx_set_error(AGX_E_INVALID, "joint_wrench and dof_force must be 16-byte aligned");
    AgxJointEffort none = {};  // no effort DOF: every joint is stepped as agx_hp1_articulated_step steps it
    const auto kern =
        art_instantiation(cfg->num_motors, art->num_bodies, [](auto m, auto nb) { return articulated_step_joint_force_kernel<m, nb>; });
    const size_t smem = sizeof(float) * kArtThreads * joint_force_row_stride(art->num_bodies);  // <= 56.8 KB at 16 bodies
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return agx_set_error(AGX_E_CUDA, "cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    }
    kern<<<art_blocks(cfg), kArtThreads, smem, (cudaStream_t)stream>>>(*cfg, *buf, *art, effort ? *effort : none, imu_body, imu_input,
                                                                       joint_wrench, dof_force);
    return agx_check_launch("articulated_step_joint_force_kernel");
}
