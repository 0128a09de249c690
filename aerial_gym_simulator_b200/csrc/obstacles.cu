// agx_obstacle_step: kinematic advance of the obstacles of the "dynamic_env" environment (env_manager/obstacle_manager.py:40-44 +
// the PhysX motion the reference relies on) -- one thread per obstacle row, arithmetic in obstacle_core.cuh (our spec, DESIGN 1 row f2').
// agx_obstacle_ground_contact: the free obstacles against the ground plane -- one thread per obstacle row, arithmetic in
// contact_core.cuh (obstacle_ground_row; DESIGN.md "Ground contact of free obstacles").
// agx_obstacle_obstacle_contact: the free obstacles against each other -- one warp per env, arithmetic in contact_core.cuh
// (obstacle_box_pair, obstacle_contacts_solve; DESIGN.md "Contact between free obstacles").
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

// One warp (= one CTA) per env.  Shared memory: the env's bodies B[A] and world boxes X[A], the contact list L[AGX_OBSTACLE_MAX_CONTACTS]
// and one AGX_CONTACT_MAX scratch per lane.  Lanes take the pairs (i, j), i < j, in order, 32 at a time (broad and narrow phase);
// a warp scan appends each round's contacts to L in pair order.  Lane 0 runs the solve, then the lanes write the touched free rows.
constexpr int kPairWarp = 32;

inline size_t obstacle_pair_smem(int A) {
    return (size_t)A * (sizeof(ContactBody) + sizeof(ObstacleBox) + 1) + sizeof(ObstacleContact) * AGX_OBSTACLE_MAX_CONTACTS +
           sizeof(ContactPt) * AGX_CONTACT_MAX * kPairWarp;
}

__global__ void __launch_bounds__(kPairWarp)
obstacle_obstacle_contact_kernel(int A, const __grid_constant__ AgxContactParams P, float* __restrict__ state, int stride,
                                 const AgxObstacleMass* __restrict__ mass, const __grid_constant__ AgxObstacleBoxes bx) {
    extern __shared__ float4 smem_raw[];
    ContactBody* B = reinterpret_cast<ContactBody*>(smem_raw);
    ObstacleContact* L = reinterpret_cast<ObstacleContact*>(B + A);
    ObstacleBox* X = reinterpret_cast<ObstacleBox*>(L + AGX_OBSTACLE_MAX_CONTACTS);
    ContactPt* S = reinterpret_cast<ContactPt*>(X + A);
    unsigned char* touched = reinterpret_cast<unsigned char*>(S + AGX_CONTACT_MAX * kPairWarp);
    const int lane = threadIdx.x;
    const long long e0 = (long long)blockIdx.x * A;
    float* rows = state + e0 * stride;
    for (int a = lane; a < A; a += kPairWarp) {
        const float* row = rows + (size_t)a * stride;
        contact_body_load(B[a], row, mass[e0 + a]);
        obstacle_box_world(row, bx.boxes + (size_t)15 * bx.asset_file[e0 + a], X[a]);
        touched[a] = 0;
    }
    __syncwarp();
    // pair index p = base + lane as (i, j): row i holds j = i+1 .. A-1
    int i = 0, j = 1 + lane;
    while (i < A - 1 && j >= A) {
        j = j - A + i + 2;
        ++i;
    }
    int count = 0;
    ContactPt* mine = S + AGX_CONTACT_MAX * lane;
    for (int base = 0; base < A * (A - 1) / 2; base += kPairWarp) {
        int n = 0;
        if (i < A - 1 && (B[i].free || B[j].free) && obstacle_box_near(P, X[i], X[j])) n = obstacle_box_pair(P, X[i], X[j], mine);
        int incl = n;
        for (int off = 1; off < kPairWarp; off <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, incl, off);
            if (lane >= off) incl += t;
        }
        const bool fits = count + incl <= AGX_OBSTACLE_MAX_CONTACTS;
        if (fits)
            for (int k = 0; k < n; ++k) {
                ObstacleContact& o = L[count + incl - n + k];
                o.c = mine[k];
                o.i = i;
                o.j = j;
            }
        const bool full = __any_sync(0xffffffffu, n > 0 && !fits);
        count += __reduce_max_sync(0xffffffffu, fits ? (unsigned)incl : 0u);
        if (full) break;
        j += kPairWarp;
        while (i < A - 1 && j >= A) {
            j = j - A + i + 2;
            ++i;
        }
    }
    __syncwarp();
    if (count == 0) return;
    if (lane == 0) {
        obstacle_contacts_solve(P, B, L, count);
        for (int q = 0; q < count; ++q) touched[L[q].i] = touched[L[q].j] = 1;
    }
    __syncwarp();
    for (int a = lane; a < A; a += kPairWarp)
        if (touched[a] && B[a].free) contact_body_store(B[a], rows + (size_t)a * stride, P.dt);
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

extern "C" int agx_obstacle_obstacle_contact(int num_envs, int num_assets, const AgxContactParams* params, float* asset_state,
                                             int asset_stride, const AgxObstacleMass* mass, const AgxObstacleBoxes* boxes, void* stream) {
    if (num_envs < 0 || num_assets < 0) return agx_set_error(AGX_E_INVALID, "agx_obstacle_obstacle_contact: negative size");
    if (num_assets > AGX_OBSTACLE_MAX_ASSETS)
        return agx_set_error(AGX_E_INVALID, "agx_obstacle_obstacle_contact: num_assets > AGX_OBSTACLE_MAX_ASSETS");
    if (asset_stride < 13) return agx_set_error(AGX_E_INVALID, "agx_obstacle_obstacle_contact: asset_stride < 13");
    if (!params || !mass || !boxes) return agx_set_error(AGX_E_NULL, "agx_obstacle_obstacle_contact: params/mass/boxes is NULL");
    if (!boxes->boxes || !boxes->asset_file) return agx_set_error(AGX_E_NULL, "agx_obstacle_obstacle_contact: a box table is NULL");
    if (boxes->num_files < 1) return agx_set_error(AGX_E_INVALID, "agx_obstacle_obstacle_contact: num_files < 1");
    const AgxContactParams& p = *params;
    if (!(p.contact_offset >= 0.0f) || !(p.dt > 0.0f) || !(p.friction >= 0.0f) || !(p.max_depenetration_velocity >= 0.0f) ||
        p.iterations < 0)
        return agx_set_error(AGX_E_INVALID, "agx_obstacle_obstacle_contact: contact params out of range");
    if (num_envs == 0 || num_assets < 2) return AGX_OK;
    if (!asset_state) return agx_set_error(AGX_E_NULL, "agx_obstacle_obstacle_contact: asset_state is NULL");
    obstacle_obstacle_contact_kernel<<<num_envs, kPairWarp, obstacle_pair_smem(num_assets), (cudaStream_t)stream>>>(
        num_assets, p, asset_state, asset_stride, mass, *boxes);
    return agx_check_launch("obstacle_obstacle_contact_kernel");
}
