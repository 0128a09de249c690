// TEST INFRASTRUCTURE ONLY -- CPU shadow of the articulated-multirotor step (aerial_gym_simulator_b200/csrc/articulated_core.cuh).
//
// Compiled as HOST code (-DAGX_HOST_SHADOW, -ffp-contract=off) like the other shadows, so tests/test_articulated_cpu.py can hold the
// kernel's own arithmetic against oracle/articulated_oracle.py without a GPU, and tests/_cpu_stack.py can run an EnvManager with an
// articulated robot on the CPU.  Nothing in the product loads this library.
#include <stdint.h>

#include "../../aerial_gym_simulator_b200/csrc/articulated_core.cuh"

using namespace agx;

template <int M, int NB>
static void sh_art_step(const AgxHp1Config& cfg, const AgxHp1Buffers& buf, const AgxArticulation& art) {
    for (int env = 0; env < cfg.num_envs; ++env) art_env_step<M, NB>(cfg, buf, art, env);  // = articulated_step_kernel<M, NB>
}

extern "C" {

// = agx_hp1_articulated_step without the argument checks (pick_art_kernel's choice of the scratch size)
int shadow_art_step(const AgxHp1Config* cfg, const AgxHp1Buffers* buf, const AgxArticulation* art) {
    const bool small = art->num_bodies <= 9;
    if (cfg->num_motors == 4) small ? sh_art_step<4, 9>(*cfg, *buf, *art) : sh_art_step<4, AGX_ART_MAX_BODIES>(*cfg, *buf, *art);
    else small ? sh_art_step<8, 9>(*cfg, *buf, *art) : sh_art_step<8, AGX_ART_MAX_BODIES>(*cfg, *buf, *art);
    return 0;
}

// art_dynamics alone.  root [13] (x, q xyzw, v, w), q / qd / qs / qds [D], grav [3], thrust [M], F_w / T_w [3];
// out: a0 [6] (spatial acceleration at the base origin, angular first), qdd [D]
void shadow_art_dynamics(const AgxArticulation* art, const float* root, const float* q, const float* qd, const float* qs, const float* qds,
                         float dt, const float* grav, int M, const float* thrust, const float* F_w, const float* T_w, float* a0, float* qdd) {
    const EnvState s = unpack(root);
    art_dynamics<AGX_ART_MAX_BODIES>(*art, s, q, qd, qs, qds, dt, ld3(grav), M, thrust, ld3(F_w), ld3(T_w), a0, qdd);
}

}  // extern "C"
