// TEST INFRASTRUCTURE ONLY -- CPU shadow of the prismatic-joint kernels of aerial_gym_simulator_b200/csrc/articulated_prismatic.cu:
// the step and the per-body state, art_env_step / art_body_states with their PRISM flag.
//
// Compiled as HOST code (-DAGX_HOST_SHADOW, -ffp-contract=off) like tests/csrc/articulated_shadow.cu, so the CPU tests can hold the
// kernels' own arithmetic against oracle/articulated_prismatic_oracle.py without a GPU, and
// tests/_cpu_stack_articulated_prismatic.py can run an EnvManager with a sliding joint on the CPU.  Each entry is its
// agx_hp1_articulated_*_prismatic without the argument checks and the stream, with the same instantiation (art_instantiation); an
// env's loop body is its kernel's thread body.  Nothing in the product loads this library.
#include <stddef.h>
#include <stdint.h>

#include "../../aerial_gym_simulator_b200/csrc/articulated_core.cuh"

using namespace agx;

extern "C" {

// the kernel builds each env's joint-force rows in shared memory and copies a warp's span out; here they are written in place.
// NULL joint_wrench writes no joint forces.
int shadow_art_step_prismatic(const AgxHp1Config* cfg, const AgxHp1Buffers* buf, const AgxArticulation* art, uint32_t pmask,
                              const AgxJointEffort* eff, int imu_body, float* imu_input, float* joint_wrench, float* dof_force) {
    AgxJointEffort none = {};
    const AgxJointEffort* e = eff ? eff : &none;
    const int B = art->num_bodies, D = art->num_dofs;
    art_instantiation(cfg->num_motors, B, [&](auto m, auto nb) {
        for (int env = 0; env < cfg->num_envs; ++env)
            art_env_step<m, nb, true, true, true, true>(*cfg, *buf, *art, env, imu_body, imu_input, e,
                                                        joint_wrench ? joint_wrench + (size_t)env * 6 * B : nullptr,
                                                        joint_wrench ? dof_force + (size_t)env * D : nullptr, pmask);
    });
    return 0;
}

int shadow_art_body_state_prismatic(const AgxArticulation* art, uint32_t pmask, int num_envs, const float* root_state,
                                    int root_state_stride, float* body_state) {
    const int B = art->num_bodies, D = art->num_dofs;
    art_instantiation(4, B, [&](auto, auto nb) {
        for (int env = 0; env < num_envs; ++env)
            art_body_states<nb, true>(*art, root_state + (size_t)env * root_state_stride, art->dof_state + (size_t)env * 2 * D,
                                      body_state + (size_t)env * 13 * B, pmask);
    });
    return 0;
}

}  // extern "C"
