// TEST INFRASTRUCTURE ONLY -- CPU shadow of the articulated step with effort-mode joints (art_env_step<M, NB, IMU, true> of
// aerial_gym_simulator_b200/csrc/articulated_core.cuh, the arithmetic of articulated_step_effort_kernel).
//
// Compiled as HOST code (-DAGX_HOST_SHADOW, -ffp-contract=off) like the other shadows, so tests/test_articulated_effort_cpu.py can
// hold the kernel's own arithmetic against oracle/articulated_effort_oracle.py without a GPU, and tests/_cpu_stack_articulated_effort.py
// can run an EnvManager with a torque-driven joint on the CPU.  Nothing in the product loads this library.
#include <stddef.h>
#include <stdint.h>

#include "../../aerial_gym_simulator_b200/csrc/articulated_core.cuh"

using namespace agx;

template <int M, int NB, bool IMU>
static void sh_art_step_effort(const AgxHp1Config& cfg, const AgxHp1Buffers& buf, const AgxArticulation& art, const AgxJointEffort& eff,
                               int imu_body, float* imu) {
    for (int env = 0; env < cfg.num_envs; ++env) art_env_step<M, NB, IMU, true>(cfg, buf, art, env, imu_body, imu, &eff);
}

template <bool IMU>
static void sh_pick(const AgxHp1Config& cfg, const AgxHp1Buffers& buf, const AgxArticulation& art, const AgxJointEffort& eff, int imu_body,
                    float* imu) {
    const bool small = art.num_bodies <= 9;
    if (cfg.num_motors == 4)
        small ? sh_art_step_effort<4, 9, IMU>(cfg, buf, art, eff, imu_body, imu)
              : sh_art_step_effort<4, AGX_ART_MAX_BODIES, IMU>(cfg, buf, art, eff, imu_body, imu);
    else
        small ? sh_art_step_effort<8, 9, IMU>(cfg, buf, art, eff, imu_body, imu)
              : sh_art_step_effort<8, AGX_ART_MAX_BODIES, IMU>(cfg, buf, art, eff, imu_body, imu);
}

extern "C" {

// = agx_hp1_articulated_step_effort without the argument checks (its choice of the instantiation)
int shadow_art_step_effort(const AgxHp1Config* cfg, const AgxHp1Buffers* buf, const AgxArticulation* art, const AgxJointEffort* eff,
                           int imu_body, float* imu_input) {
    if (imu_input) sh_pick<true>(*cfg, *buf, *art, *eff, imu_body, imu_input);
    else sh_pick<false>(*cfg, *buf, *art, *eff, imu_body, nullptr);
    return 0;
}

}  // extern "C"
