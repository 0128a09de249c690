// TEST INFRASTRUCTURE ONLY -- CPU shadow of the dynamic-obstacle contact solve (aerial_gym_simulator_b200/csrc/contact_core.cuh,
// contact_bodies_gather and contact_env_dynamic, as hp2_contact_dynamic_kernel runs them after its contact search).
//
// Compiled as HOST code (-DAGX_HOST_SHADOW, -ffp-contract=off) like tests/csrc/contact_moving_shadow.cu, so
// tests/test_contact_dynamic_cpu.py can hold the kernel's own arithmetic against oracle/contact_dynamic_oracle.py bit for bit
// without a GPU.  Nothing in the product loads this library.
#include <stdint.h>

#include "../../aerial_gym_simulator_b200/csrc/contact_core.cuh"

using namespace agx;

extern "C" {

// contacts [E, AGX_CONTACT_MAX, 7] = point xyz, normal xyz, depth; count [E]; ids [E, AGX_CONTACT_MAX] (object index, K = ground);
// asset_state [E, A, stride] (read and written), obj_asset [E, K], mass [E, A]
void shadow_contact_solve_dynamic(int num_envs, const AgxContactParams* p, float* root_state, int stride, const float* contacts,
                                  const int32_t* count, const int32_t* ids, int K, float* asset_state, int A, int asset_stride,
                                  const int32_t* obj_asset, const AgxObstacleMass* mass, float* force, uint8_t* crashes) {
    for (int e = 0; e < num_envs; ++e) {
        ContactPt c[AGX_CONTACT_MAX];
        int id[AGX_CONTACT_MAX];
        const int n = count[e];
        for (int i = 0; i < n; ++i) {
            const float* s = contacts + ((size_t)e * AGX_CONTACT_MAX + i) * 7;
            c[i] = ContactPt{{s[0], s[1], s[2]}, {s[3], s[4], s[5]}, s[6]};
            id[i] = ids[(size_t)e * AGX_CONTACT_MAX + i];
        }
        float* f = force + (size_t)e * 3;
        if (n == 0) {
            f[0] = f[1] = f[2] = 0.0f;
            continue;
        }
        ContactBody B[AGX_CONTACT_MAX];
        float* rows[AGX_CONTACT_MAX];
        int body[AGX_CONTACT_MAX];
        const int nb = contact_bodies_gather(id, n, K, obj_asset + (size_t)e * K, asset_state + (size_t)e * A * asset_stride, asset_stride,
                                             mass + (size_t)e * A, B, rows, body);
        contact_env_dynamic(*p, root_state + (size_t)e * stride, c, n, f, crashes + e, body, B, nb, rows);
    }
}

}  // extern "C"
