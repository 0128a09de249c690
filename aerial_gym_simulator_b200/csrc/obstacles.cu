// agx_obstacle_step: kinematic advance of the obstacles of the "dynamic_env" environment (env_manager/obstacle_manager.py:40-44 +
// the PhysX motion the reference relies on) -- one thread per obstacle row, arithmetic in obstacle_core.cuh (our spec, DESIGN 1 row f2').
// agx_obstacle_ground_contact: the free obstacles against the ground plane -- one thread per obstacle row, arithmetic in
// contact_core.cuh (obstacle_ground_row; DESIGN.md "Ground contact of free obstacles").
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/aerial_gym_b200.h"
#include "agx_common.cuh"
#include "contact_core.cuh"
#include "obstacle_core.cuh"

namespace {
using namespace agx;
constexpr int kEnvThreads = 128;

__global__ void __launch_bounds__(kEnvThreads)
obstacle_step_kernel(long long total, float* __restrict__ state, int stride, const float* __restrict__ twist, float dt, int substeps,
                     float lin_damp, float ang_damp) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    obstacle_step_item(i, state, stride, twist, dt, substeps, lin_damp, ang_damp);
}

// row i = (env, asset) of the [E,A] tables; no scene, no shared memory
__global__ void __launch_bounds__(kEnvThreads)
obstacle_ground_contact_kernel(long long total, const __grid_constant__ AgxContactParams P, float* __restrict__ state, int stride,
                               const AgxObstacleMass* __restrict__ mass, const __grid_constant__ AgxObstacleHull h) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int f = h.asset_file[i];
    const int v0 = h.file_offset[f];
    obstacle_ground_row(P, state + i * stride, mass[i], h.vertices + (size_t)3 * v0, h.file_offset[f + 1] - v0, h.file_reach[f], nullptr);
}

inline int blocks_for(long long n) { return (int)((n + kEnvThreads - 1) / kEnvThreads); }
}  // namespace

extern "C" int agx_obstacle_step(int num_envs, int num_assets, float* asset_state, int asset_stride, const float* twist, float dt, int substeps,
                      float linear_damping, float angular_damping, void* stream) {
    if (num_envs < 0 || num_assets < 0 || substeps < 0) return agx_set_error(AGX_E_INVALID, "agx_obstacle_step: negative size");
    if (asset_stride < 13) return agx_set_error(AGX_E_INVALID, "agx_obstacle_step: asset_stride < 13");
    if (!(dt > 0.0f)) return agx_set_error(AGX_E_INVALID, "agx_obstacle_step: dt must be > 0");
    const long long total = (long long)num_envs * num_assets;
    if (total == 0 || substeps == 0) return AGX_OK;
    if (!asset_state) return agx_set_error(AGX_E_NULL, "agx_obstacle_step: asset_state is NULL");
    obstacle_step_kernel<<<blocks_for(total), kEnvThreads, 0, (cudaStream_t)stream>>>(total, asset_state, asset_stride, twist, dt, substeps,
                                                                                      linear_damping, angular_damping);
    return agx_check_launch("obstacle_step_kernel");
}

extern "C" int agx_obstacle_ground_contact(int num_envs, int num_assets, const AgxContactParams* params, float* asset_state,
                                           int asset_stride, const AgxObstacleMass* mass, const AgxObstacleHull* hull, void* stream) {
    if (num_envs < 0 || num_assets < 0) return agx_set_error(AGX_E_INVALID, "agx_obstacle_ground_contact: negative size");
    if (asset_stride < 13) return agx_set_error(AGX_E_INVALID, "agx_obstacle_ground_contact: asset_stride < 13");
    if (!params || !mass || !hull) return agx_set_error(AGX_E_NULL, "agx_obstacle_ground_contact: params/mass/hull is NULL");
    if (!hull->vertices || !hull->file_offset || !hull->file_reach || !hull->asset_file)
        return agx_set_error(AGX_E_NULL, "agx_obstacle_ground_contact: a hull table is NULL");
    if (hull->num_files < 1) return agx_set_error(AGX_E_INVALID, "agx_obstacle_ground_contact: num_files < 1");
    const AgxContactParams& p = *params;
    if (!(p.contact_offset >= 0.0f) || !(p.dt > 0.0f) || !(p.friction >= 0.0f) || !(p.max_depenetration_velocity >= 0.0f) ||
        p.iterations < 0)
        return agx_set_error(AGX_E_INVALID, "agx_obstacle_ground_contact: contact params out of range");
    const long long total = (long long)num_envs * num_assets;
    if (total == 0) return AGX_OK;
    if (!asset_state) return agx_set_error(AGX_E_NULL, "agx_obstacle_ground_contact: asset_state is NULL");
    obstacle_ground_contact_kernel<<<blocks_for(total), kEnvThreads, 0, (cudaStream_t)stream>>>(total, p, asset_state, asset_stride,
                                                                                               mass, *hull);
    return agx_check_launch("obstacle_ground_contact_kernel");
}
