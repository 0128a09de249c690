// TEST INFRASTRUCTURE ONLY -- CPU shadow of the articulated-multirotor kernels (aerial_gym_simulator_b200/csrc/articulated_core.cuh):
// the step in its four variants (plain, IMU, effort, joint forces), the per-body state, and art_dynamics alone.
//
// Compiled as HOST code (-DAGX_HOST_SHADOW, -ffp-contract=off) like the other shadows, so the CPU tests can hold the kernels' own
// arithmetic against the float64 oracles under oracle/ without a GPU, and tests/_cpu_stack_articulated.py can run an EnvManager with
// an articulated robot on the CPU.  Each shadow_art_step* entry is its agx_hp1_articulated_step* without the argument checks and the
// stream, with the same instantiation (art_instantiation); an env's loop body is its kernel's thread body.  Nothing in the product
// loads this library.
#include <stddef.h>
#include <stdint.h>

#include "../../aerial_gym_simulator_b200/csrc/articulated_core.cuh"

using namespace agx;

extern "C" {

int shadow_art_step(const AgxHp1Config* cfg, const AgxHp1Buffers* buf, const AgxArticulation* art) {
    art_instantiation(cfg->num_motors, art->num_bodies, [&](auto m, auto nb) {
        for (int env = 0; env < cfg->num_envs; ++env) art_env_step<m, nb>(*cfg, *buf, *art, env);
    });
    return 0;
}

int shadow_art_step_imu(const AgxHp1Config* cfg, const AgxHp1Buffers* buf, const AgxArticulation* art, int imu_body, float* imu_input) {
    art_instantiation(cfg->num_motors, art->num_bodies, [&](auto m, auto nb) {
        for (int env = 0; env < cfg->num_envs; ++env) art_env_step<m, nb, true>(*cfg, *buf, *art, env, imu_body, imu_input);
    });
    return 0;
}

int shadow_art_step_effort(const AgxHp1Config* cfg, const AgxHp1Buffers* buf, const AgxArticulation* art, const AgxJointEffort* eff,
                           int imu_body, float* imu_input) {
    art_instantiation(cfg->num_motors, art->num_bodies, [&](auto m, auto nb) {
        for (int env = 0; env < cfg->num_envs; ++env) {
            if (imu_input) art_env_step<m, nb, true, true>(*cfg, *buf, *art, env, imu_body, imu_input, eff);
            else art_env_step<m, nb, false, true>(*cfg, *buf, *art, env, imu_body, nullptr, eff);
        }
    });
    return 0;
}

// the kernel builds each env's rows in shared memory and copies a warp's span out; here they are written in place
int shadow_art_step_joint_force(const AgxHp1Config* cfg, const AgxHp1Buffers* buf, const AgxArticulation* art, const AgxJointEffort* eff,
                                int imu_body, float* imu_input, float* joint_wrench, float* dof_force) {
    AgxJointEffort none = {};
    const AgxJointEffort* e = eff ? eff : &none;
    const int B = art->num_bodies, D = art->num_dofs;
    art_instantiation(cfg->num_motors, B, [&](auto m, auto nb) {
        for (int env = 0; env < cfg->num_envs; ++env)
            art_env_step<m, nb, true, true, true>(*cfg, *buf, *art, env, imu_body, imu_input, e, joint_wrench + (size_t)env * 6 * B,
                                                  dof_force + (size_t)env * D);
    });
    return 0;
}

// the kernel builds each env's rows in shared memory and copies a warp's span out; here they are built in place in the output
int shadow_art_body_state(const AgxArticulation* art, int num_envs, const float* root_state, int root_state_stride, float* body_state) {
    const int B = art->num_bodies, D = art->num_dofs;
    art_instantiation(4, B, [&](auto, auto nb) {
        for (int env = 0; env < num_envs; ++env)
            art_body_states<nb>(*art, root_state + (size_t)env * root_state_stride, art->dof_state + (size_t)env * 2 * D,
                                body_state + (size_t)env * 13 * B);
    });
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
