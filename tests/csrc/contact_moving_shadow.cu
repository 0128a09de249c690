// TEST INFRASTRUCTURE ONLY -- CPU shadow of the moving-obstacle contact solve (aerial_gym_simulator_b200/csrc/contact_core.cuh,
// contact_solve<true> and obstacle_point_vel, as hp2_contact_moving_kernel runs them).
//
// Compiled as HOST code (-DAGX_HOST_SHADOW, -ffp-contract=off) like tests/csrc/contact_shadow.cu, so tests/test_contact_moving_cpu.py
// can hold the kernel's own arithmetic against oracle/contact_moving_oracle.py bit for bit without a GPU.  Nothing in the product
// loads this library.
#include <stdint.h>

#include "../../aerial_gym_simulator_b200/csrc/contact_core.cuh"

using namespace agx;

extern "C" {

// contacts [E, AGX_CONTACT_MAX, 7] = point xyz, normal xyz, depth; count [E]; u [E, AGX_CONTACT_MAX, 3] obstacle point velocities
void shadow_contact_solve_moving(int num_envs, const AgxContactParams* p, float* root_state, int stride, const float* contacts,
                                 const int32_t* count, const float* u, float* force, uint8_t* crashes) {
    for (int e = 0; e < num_envs; ++e) {
        ContactPt c[AGX_CONTACT_MAX];
        float ue[AGX_CONTACT_MAX][3];
        const int n = count[e];
        for (int i = 0; i < n; ++i) {
            const float* s = contacts + ((size_t)e * AGX_CONTACT_MAX + i) * 7;
            c[i] = ContactPt{{s[0], s[1], s[2]}, {s[3], s[4], s[5]}, s[6]};
            for (int k = 0; k < 3; ++k) ue[i][k] = u[((size_t)e * AGX_CONTACT_MAX + i) * 3 + k];
        }
        float* f = force + (size_t)e * 3;
        if (n == 0) {
            f[0] = f[1] = f[2] = 0.0f;
            continue;
        }
        contact_env<true>(*p, root_state + (size_t)e * stride, c, n, f, crashes + e, ue);
    }
}

// u of one contact point p from an asset row (x y z q v w)
void shadow_obstacle_point_vel(const float* row, const float* p, float* u) { obstacle_point_vel(row, p, u); }

}  // extern "C"
