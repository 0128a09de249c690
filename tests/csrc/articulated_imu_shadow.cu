// TEST INFRASTRUCTURE ONLY -- CPU shadow of the articulated step with the IMU input of one body (art_env_step<M, NB, true> of
// aerial_gym_simulator_b200/csrc/articulated_core.cuh, the arithmetic of articulated_step_imu_kernel).
//
// Compiled as HOST code (-DAGX_HOST_SHADOW, -ffp-contract=off) like the other shadows, so tests/test_articulated_imu_cpu.py can hold
// the kernel's own arithmetic against oracle/articulated_imu_oracle.py without a GPU, and tests/_cpu_stack_articulated_imu.py can run
// an EnvManager with an IMU on a link on the CPU.  Nothing in the product loads this library.
#include <stddef.h>
#include <stdint.h>

#include "../../aerial_gym_simulator_b200/csrc/articulated_core.cuh"

using namespace agx;

template <int M, int NB>
static void sh_art_step_imu(const AgxHp1Config& cfg, const AgxHp1Buffers& buf, const AgxArticulation& art, int imu_body, float* imu) {
    for (int env = 0; env < cfg.num_envs; ++env) art_env_step<M, NB, true>(cfg, buf, art, env, imu_body, imu);
}

extern "C" {

// = agx_hp1_articulated_step_imu without the argument checks (its choice of the instantiation)
int shadow_art_step_imu(const AgxHp1Config* cfg, const AgxHp1Buffers* buf, const AgxArticulation* art, int imu_body, float* imu_input) {
    const bool small = art->num_bodies <= 9;
    if (cfg->num_motors == 4)
        small ? sh_art_step_imu<4, 9>(*cfg, *buf, *art, imu_body, imu_input)
              : sh_art_step_imu<4, AGX_ART_MAX_BODIES>(*cfg, *buf, *art, imu_body, imu_input);
    else
        small ? sh_art_step_imu<8, 9>(*cfg, *buf, *art, imu_body, imu_input)
              : sh_art_step_imu<8, AGX_ART_MAX_BODIES>(*cfg, *buf, *art, imu_body, imu_input);
    return 0;
}

}  // extern "C"
