// Articulated multirotors with prismatic joints (DESIGN.md "Articulated robots", "Prismatic joints"): the step and the per-body
// state of a robot whose tree mixes revolute, continuous and prismatic joints.  The joint kind of each body is read at run time from
// a bit mask, so one robot can mix them; the per-env arithmetic is articulated_core.cuh's with its PRISM flag.  A unit of its own:
// the kernels of articulated.cu keep their machine code.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/aerial_gym_b200.h"
#include "agx_common.cuh"
#include "articulated_core.cuh"
#include "articulated_launch.cuh"

using namespace agx;

namespace {

// ---- the step (agx_hp1_articulated_step_prismatic): the joint-force kernel's arithmetic and layout, with the joint kinds of
// prismatic_mask.  The IMU input (NULL imu_input), the effort DOFs (a table without effort DOFs) and the joint forces (NULL
// joint_wrench) are resolved at run time, so four instantiations cover every robot; without the joint forces the launch has no
// shared memory and nothing is copied out.
template <int M, int NB>
__global__ void __launch_bounds__(kArtThreads)
articulated_step_prismatic_kernel(const __grid_constant__ AgxHp1Config cfg, const __grid_constant__ AgxHp1Buffers buf,
                                  const __grid_constant__ AgxArticulation art, uint32_t prismatic_mask,
                                  const __grid_constant__ AgxJointEffort eff, int imu_body, float* __restrict__ imu_input,
                                  float* __restrict__ joint_wrench, float* __restrict__ dof_force) {
    extern __shared__ float s_joint_rows[];
    const int lane = threadIdx.x % kWarp;
    const int env0 = blockIdx.x * blockDim.x + threadIdx.x - lane;
    if (env0 >= cfg.num_envs) return;  // whole warps only: the rest of the warp copies below
    const int B = art.num_bodies, D = art.num_dofs, W = 6 * B, st = joint_force_row_stride(B);
    float* s_warp = s_joint_rows + (threadIdx.x - lane) * st;
    const int env = env0 + lane;
    const bool jf = joint_wrench != nullptr;
    if (env < cfg.num_envs)
        art_env_step<M, NB, true, true, true, true>(cfg, buf, art, env, imu_body, imu_input, &eff, jf ? s_warp + lane * st : nullptr,
                                                    jf ? s_warp + lane * st + W : nullptr, prismatic_mask);
    if (!jf) return;
    __syncwarp();
    const int n = min(kWarp, cfg.num_envs - env0);
    copy_warp_rows(joint_wrench + (size_t)env0 * W, s_warp, st, 0, W, n, lane);  // 16-byte aligned: env0 W is a multiple of 32 x 6
    if (D) copy_warp_rows(dof_force + (size_t)env0 * D, s_warp, st, W, D, n, lane);
}

// ---- per-body state (agx_hp1_articulated_body_state_prismatic): articulated_body_state_kernel's layout -- one env per lane, its
// rows built in shared memory (13 B floats, made odd) and the warp's contiguous span copied out with 16-byte stores
template <int NB>
__global__ void __launch_bounds__(kBodyThreads)
articulated_body_state_prismatic_kernel(const __grid_constant__ AgxArticulation art, uint32_t prismatic_mask, int num_envs,
                                        const float* __restrict__ root_state, int root_stride, float* __restrict__ body_state) {
    extern __shared__ float s_rows[];
    const int B = art.num_bodies, D = art.num_dofs;
    const int len = 13 * B, st = len | 1;
    const int lane = threadIdx.x;
    const int env0 = blockIdx.x * kBodyThreads;
    const int env = env0 + lane;
    if (env < num_envs)
        art_body_states<NB, true>(art, root_state + (size_t)env * root_stride, art.dof_state + (size_t)env * 2 * D, s_rows + lane * st,
                                  prismatic_mask);
    __syncwarp();
    // 16-byte aligned: env0 len is a multiple of 32 x 13
    copy_warp_rows(body_state + (size_t)env0 * len, s_rows, st, 0, len, min(kBodyThreads, num_envs - env0), lane);
}

// the joint kinds: body 0 is the base, bits past the tree name no body, and every slide is bounded (its projection keeps each body
// within the robot's size of the base origin, what the float32 arithmetic rests on)
int validate_prismatic(const AgxArticulation* art, uint32_t mask) {
    if (mask & 1u) return agx_set_error(AGX_E_INVALID, "prismatic_mask bit 0 is set: body 0 is the floating base and has no joint");
    if (art->num_bodies < 32 && (mask >> art->num_bodies))
        return agx_set_error(AGX_E_INVALID, "prismatic_mask has bits at or above num_bodies = %d", art->num_bodies);
    for (int i = 1; i < art->num_bodies; ++i)
        if (((mask >> i) & 1u) && !(art->limited[i] && art->lower[i] < art->upper[i]))
            return agx_set_error(AGX_E_INVALID, "body %d's joint is prismatic: it must be limited, with lower < upper", i);
    return AGX_OK;
}

}  // namespace

extern "C" int agx_hp1_articulated_step_prismatic(const AgxHp1Config* cfg, const AgxHp1Buffers* buf, const AgxArticulation* art,
                                                  uint32_t prismatic_mask, const AgxJointEffort* effort, int imu_body, float* imu_input,
                                                  float* joint_wrench, float* dof_force, void* stream) {
    int rc = validate_step(cfg, buf, art, effort, imu_input != nullptr, imu_body);
    if (rc) return rc;
    if ((rc = validate_prismatic(art, prismatic_mask))) return rc;
    if (cfg->num_envs == 0) return AGX_OK;
    if (!joint_wrench && dof_force) return agx_set_error(AGX_E_INVALID, "dof_force is given without joint_wrench: pass both or neither");
    if (joint_wrench && art->num_dofs > 0 && !dof_force) return agx_set_error(AGX_E_NULL, "dof_force is NULL and joint_wrench is not");
    if (((uintptr_t)joint_wrench | (uintptr_t)dof_force) & 15)
        return agx_set_error(AGX_E_INVALID, "joint_wrench and dof_force must be 16-byte aligned");
    AgxJointEffort none = {};  // no effort DOF: every joint is driven by its implicit drive
    const auto kern =
        art_instantiation(cfg->num_motors, art->num_bodies, [](auto m, auto nb) { return articulated_step_prismatic_kernel<m, nb>; });
    const size_t smem = joint_wrench ? sizeof(float) * kArtThreads * joint_force_row_stride(art->num_bodies) : 0;  // <= 56.8 KB
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return agx_set_error(AGX_E_CUDA, "cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    }
    kern<<<art_blocks(cfg), kArtThreads, smem, (cudaStream_t)stream>>>(*cfg, *buf, *art, prismatic_mask, effort ? *effort : none,
                                                                       imu_body, imu_input, joint_wrench, dof_force);
    return agx_check_launch("articulated_step_prismatic_kernel");
}

extern "C" int agx_hp1_articulated_body_state_prismatic(const AgxArticulation* art, uint32_t prismatic_mask, int num_envs,
                                                        const float* root_state, int root_state_stride, float* body_state, void* stream) {
    int rc = validate_body_state(art, num_envs, root_state, root_state_stride, body_state);
    if (rc) return rc;
    if ((rc = validate_prismatic(art, prismatic_mask))) return rc;
    if (num_envs == 0) return AGX_OK;
    const int g = (num_envs + kBodyThreads - 1) / kBodyThreads;
    const size_t smem = sizeof(float) * kBodyThreads * ((13 * art->num_bodies) | 1);  // <= 26.75 KB at 16 bodies
    // the kernel has no motors: only the tree size of the instantiation applies
    const auto kern = art_instantiation(4, art->num_bodies, [](auto, auto nb) { return articulated_body_state_prismatic_kernel<nb>; });
    kern<<<g, kBodyThreads, smem, (cudaStream_t)stream>>>(*art, prismatic_mask, num_envs, root_state, root_state_stride, body_state);
    return agx_check_launch("articulated_body_state_prismatic_kernel");
}
