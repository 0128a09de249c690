// TEST INFRASTRUCTURE ONLY -- CPU shadow of the per-body state of an articulated robot (art_body_states of
// aerial_gym_simulator_b200/csrc/articulated_core.cuh, the arithmetic of articulated_body_state_kernel).
//
// Compiled as HOST code (-DAGX_HOST_SHADOW, -ffp-contract=off) like the other shadows.  The kernel builds each env's rows in shared
// memory and copies a warp's span out; here each env's rows are built in place in the output.  Nothing in the product loads this
// library.
#include <stddef.h>
#include <stdint.h>

#include "../../aerial_gym_simulator_b200/csrc/articulated_core.cuh"

using namespace agx;

template <int NB>
static void sh_body_state(const AgxArticulation& art, int num_envs, const float* root, int stride, float* out) {
    const int B = art.num_bodies, D = art.num_dofs;
    for (int env = 0; env < num_envs; ++env)
        art_body_states<NB>(art, root + (size_t)env * stride, art.dof_state + (size_t)env * 2 * D, out + (size_t)env * 13 * B);
}

extern "C" {

// = agx_hp1_articulated_body_state without the argument checks (its choice of the tree size)
int shadow_art_body_state(const AgxArticulation* art, int num_envs, const float* root_state, int root_state_stride, float* body_state) {
    if (art->num_bodies <= 9) sh_body_state<9>(*art, num_envs, root_state, root_state_stride, body_state);
    else sh_body_state<AGX_ART_MAX_BODIES>(*art, num_envs, root_state, root_state_stride, body_state);
    return 0;
}

}  // extern "C"
