// TEST INFRASTRUCTURE ONLY -- CPU shadow of the contact solve (aerial_gym_simulator_b200/csrc/contact_core.cuh).
//
// The solve epilogue of hp2_contact_kernel compiled a second time as HOST code (-DAGX_HOST_SHADOW, -ffp-contract=off) and driven by
// a loop over envs, so tests/test_contact_cpu.py can hold the kernel's own arithmetic against oracle/contact_oracle.py bit for bit
// on a machine without a GPU.  Nothing in the product loads this library.
#include <stdint.h>

#include "../../aerial_gym_simulator_b200/csrc/contact_core.cuh"

using namespace agx;

extern "C" {

// contacts [E, AGX_CONTACT_MAX, 7] = point xyz, normal xyz, depth; count [E]
void shadow_contact_solve(int num_envs, const AgxContactParams* p, float* root_state, int stride, const float* contacts,
                          const int32_t* count, float* force, uint8_t* crashes) {
    for (int e = 0; e < num_envs; ++e) {
        ContactPt c[AGX_CONTACT_MAX];
        const int n = count[e];
        for (int i = 0; i < n; ++i) {
            const float* s = contacts + ((size_t)e * AGX_CONTACT_MAX + i) * 7;
            c[i] = ContactPt{{s[0], s[1], s[2]}, {s[3], s[4], s[5]}, s[6]};
        }
        float* f = force + (size_t)e * 3;
        if (n == 0) {
            f[0] = f[1] = f[2] = 0.0f;
            continue;
        }
        contact_env(*p, root_state + (size_t)e * stride, c, n, f, crashes + e);
    }
}

// contact_insert, fed in the given order: returns the kept count, ids in out_id
int shadow_contact_select(int n_in, const float* key, const int32_t* obj, int32_t* out_id) {
    ContactPt c[AGX_CONTACT_MAX], pt{};
    float k[AGX_CONTACT_MAX];
    int id[AGX_CONTACT_MAX];
    int n = 0;
    for (int i = 0; i < n_in; ++i) n = contact_insert(c, k, id, n, pt, key[i], obj[i]);
    for (int i = 0; i < n; ++i) out_id[i] = id[i];
    return n;
}

}  // extern "C"
