// The launch side the articulated step units share (articulated.cu, articulated_prismatic.cu): block sizes, the argument checks of
// their entries, and the warp's copy of its lanes' rows out of shared memory.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/aerial_gym_b200.h"
#include "agx_common.cuh"

namespace {

constexpr int kArtThreads = 128;

// one env per lane, one warp per block (the body-state kernels)
constexpr int kBodyThreads = 32;

int validate_articulation(const AgxHp1Config* cfg, const AgxHp1Buffers* buf, const AgxArticulation* art) {
    if (!cfg || !buf || !art) return agx_set_error(AGX_E_NULL, "cfg/buf/art is NULL");
    if (cfg->num_envs < 0) return agx_set_error(AGX_E_INVALID, "num_envs < 0");
    if (cfg->num_motors != 4 && cfg->num_motors != 8)
        return agx_set_error(AGX_E_INVALID, "num_motors must be 4 or 8 (got %d)", cfg->num_motors);
    if (cfg->controller < AGX_CTRL_NONE || cfg->controller > AGX_CTRL_VELOCITY_STEERING)
        return agx_set_error(AGX_E_INVALID, "unknown controller id %d", cfg->controller);
    const int need = (cfg->controller == AGX_CTRL_NONE) ? cfg->num_motors : (cfg->controller == AGX_CTRL_FULLY_ACTUATED ? 7 : 4);
    if (cfg->num_actions != need)
        return agx_set_error(AGX_E_INVALID, "controller %d needs %d action columns (got %d)", cfg->controller, need, cfg->num_actions);
    if (cfg->physics_steps < 0) return agx_set_error(AGX_E_INVALID, "physics_steps < 0");
    const int B = art->num_bodies;
    if (B < 1 || B > AGX_ART_MAX_BODIES)
        return agx_set_error(AGX_E_INVALID, "num_bodies must be in [1, %d] (got %d)", AGX_ART_MAX_BODIES, B);
    if (art->num_dofs != B - 1) return agx_set_error(AGX_E_INVALID, "num_dofs must be num_bodies - 1");
    for (int i = 1; i < B; ++i)
        if (art->parent[i] < 0 || art->parent[i] >= i) return agx_set_error(AGX_E_INVALID, "parent[%d] must be in [0, %d)", i, i);
    for (int k = 0; k < cfg->num_motors; ++k)
        if (art->motor_body[k] < 0 || art->motor_body[k] >= B) return agx_set_error(AGX_E_INVALID, "motor_body[%d] out of range", k);
    if (cfg->num_envs == 0) return AGX_OK;
    if (!buf->root_state || !buf->motor_thrust || !buf->actions) return agx_set_error(AGX_E_NULL, "root_state/motor_thrust/actions is NULL");
    if (buf->body_wrench) return agx_set_error(AGX_E_INVALID, "the articulated step does not write body_wrench: pass NULL");
    if (B > 1 && (!art->dof_state || !art->dof_position_setpoint || !art->dof_velocity_setpoint))
        return agx_set_error(AGX_E_NULL, "dof_state/dof_position_setpoint/dof_velocity_setpoint is NULL");
    return AGX_OK;
}

// the checks of an effort table against art; its command array only where a DOF is in effort mode and there are envs
int validate_effort(const AgxHp1Config* cfg, const AgxArticulation* art, const AgxJointEffort* effort) {
    bool any = false;
    for (int i = 1; i < art->num_bodies; ++i) {
        if (!(effort->effort_limit[i] >= 0.0f))
            return agx_set_error(AGX_E_INVALID, "effort_limit[%d] must be >= 0 (got %g)", i, (double)effort->effort_limit[i]);
        if (!effort->effort_dof[i]) continue;
        if (art->stiffness[i] != 0.0f)
            return agx_set_error(AGX_E_INVALID, "body %d's joint is in effort mode: it has no implicit drive, stiffness[%d] must be 0", i, i);
        any = true;
    }
    if (cfg->num_envs > 0 && any && !effort->effort)
        return agx_set_error(AGX_E_NULL, "effort->effort is NULL and a joint is in effort mode");
    return AGX_OK;
}

// the checks the step entries share: the articulation, the effort table where one is given, imu_body where the IMU is written
int validate_step(const AgxHp1Config* cfg, const AgxHp1Buffers* buf, const AgxArticulation* art, const AgxJointEffort* effort,
                  bool imu, int imu_body) {
    int rc = validate_articulation(cfg, buf, art);
    if (rc) return rc;
    if (effort && (rc = validate_effort(cfg, art, effort))) return rc;
    if (imu && (imu_body < 0 || imu_body >= art->num_bodies))
        return agx_set_error(AGX_E_INVALID, "imu_body must be in [0, %d) (got %d)", art->num_bodies, imu_body);
    return AGX_OK;
}

// blocks of the step kernels: one env per thread
int art_blocks(const AgxHp1Config* cfg) { return (cfg->num_envs + kArtThreads - 1) / kArtThreads; }

int validate_body_state(const AgxArticulation* art, int num_envs, const float* root_state, int root_state_stride, const float* body_state) {
    if (!art) return agx_set_error(AGX_E_NULL, "art is NULL");
    if (num_envs < 0) return agx_set_error(AGX_E_INVALID, "num_envs < 0");
    const int B = art->num_bodies;
    if (B < 1 || B > AGX_ART_MAX_BODIES)
        return agx_set_error(AGX_E_INVALID, "num_bodies must be in [1, %d] (got %d)", AGX_ART_MAX_BODIES, B);
    if (art->num_dofs != B - 1) return agx_set_error(AGX_E_INVALID, "num_dofs must be num_bodies - 1");
    for (int i = 1; i < B; ++i)
        if (art->parent[i] < 0 || art->parent[i] >= i) return agx_set_error(AGX_E_INVALID, "parent[%d] must be in [0, %d)", i, i);
    if (root_state_stride < 13) return agx_set_error(AGX_E_INVALID, "root_state_stride < 13");
    if (num_envs == 0) return AGX_OK;
    if (!root_state || !body_state) return agx_set_error(AGX_E_NULL, "root_state/body_state is NULL");
    if (B > 1 && !art->dof_state) return agx_set_error(AGX_E_NULL, "dof_state is NULL");
    if ((uintptr_t)body_state & 15) return agx_set_error(AGX_E_INVALID, "body_state must be 16-byte aligned");
    return AGX_OK;
}

// ---- the warp's copy of its lanes' rows (the joint-force and body-state kernels) -------------------------------------------
constexpr int kWarp = 32;

// out[0, n len) = the rows [n][len] of a warp's lanes, lane e's at s + e st + off; out 16-byte aligned
__device__ void copy_warp_rows(float* __restrict__ out, const float* s, int st, int off, int len, int n, int lane) {
    const int total = n * len, n4 = total >> 2;
    for (int k = lane; k < n4; k += kWarp) {
        float v[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int g = 4 * k + j, e = g / len;
            v[j] = s[e * st + off + g - e * len];
        }
        reinterpret_cast<float4*>(out)[k] = make_float4(v[0], v[1], v[2], v[3]);
    }
    for (int g = 4 * n4 + lane; g < total; g += kWarp) {
        const int e = g / len;
        out[g] = s[e * st + off + g - e * len];
    }
}

// floats of one lane's rows in shared memory: 6 B + D, made odd
inline __host__ __device__ int joint_force_row_stride(int B) { return (7 * B - 1) | 1; }

}  // namespace
