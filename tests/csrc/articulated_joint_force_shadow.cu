// TEST INFRASTRUCTURE ONLY -- CPU shadow of the articulated step with the joint forces (art_env_step<M, NB, true, true, true> of
// aerial_gym_simulator_b200/csrc/articulated_core.cuh, the arithmetic of articulated_step_joint_force_kernel).
//
// Compiled as HOST code (-DAGX_HOST_SHADOW, -ffp-contract=off) like the other shadows, so tests/test_articulated_joint_force_cpu.py
// can hold the kernel's own arithmetic against oracle/articulated_joint_force_oracle.py without a GPU, and
// tests/_cpu_stack_articulated_joint_force.py can run an EnvManager with joint force sensing on the CPU.  Nothing in the product
// loads this library.
#include <stddef.h>
#include <stdint.h>

#include "../../aerial_gym_simulator_b200/csrc/articulated_core.cuh"

using namespace agx;

template <int M, int NB>
static void sh_art_step_joint_force(const AgxHp1Config& cfg, const AgxHp1Buffers& buf, const AgxArticulation& art,
                                    const AgxJointEffort& eff, int imu_body, float* imu, float* jw, float* dof) {
    const int B = art.num_bodies, D = art.num_dofs;
    for (int env = 0; env < cfg.num_envs; ++env)
        art_env_step<M, NB, true, true, true>(cfg, buf, art, env, imu_body, imu, &eff, jw + (size_t)env * 6 * B, dof + (size_t)env * D);
}

extern "C" {

// = agx_hp1_articulated_step_joint_force without the argument checks (its choice of the instantiation, its zeroed effort table)
int shadow_art_step_joint_force(const AgxHp1Config* cfg, const AgxHp1Buffers* buf, const AgxArticulation* art, const AgxJointEffort* eff,
                                int imu_body, float* imu_input, float* joint_wrench, float* dof_force) {
    AgxJointEffort none = {};
    const AgxJointEffort& e = eff ? *eff : none;
    const bool small = art->num_bodies <= 9;
    if (cfg->num_motors == 4)
        small ? sh_art_step_joint_force<4, 9>(*cfg, *buf, *art, e, imu_body, imu_input, joint_wrench, dof_force)
              : sh_art_step_joint_force<4, AGX_ART_MAX_BODIES>(*cfg, *buf, *art, e, imu_body, imu_input, joint_wrench, dof_force);
    else
        small ? sh_art_step_joint_force<8, 9>(*cfg, *buf, *art, e, imu_body, imu_input, joint_wrench, dof_force)
              : sh_art_step_joint_force<8, AGX_ART_MAX_BODIES>(*cfg, *buf, *art, e, imu_body, imu_input, joint_wrench, dof_force);
    return 0;
}

}  // extern "C"
