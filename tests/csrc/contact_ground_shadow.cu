// TEST INFRASTRUCTURE ONLY -- CPU shadow of the obstacle-ground contact (aerial_gym_simulator_b200/csrc/contact_core.cuh,
// obstacle_ground_row, as obstacle_ground_contact_kernel runs it per (env, asset) row).
//
// Compiled as HOST code (-DAGX_HOST_SHADOW, -ffp-contract=off) like tests/csrc/contact_dynamic_shadow.cu, so
// tests/test_contact_ground_cpu.py can hold the kernel's own arithmetic against oracle/contact_ground_oracle.py bit for bit
// without a GPU.  Nothing in the product loads this library.
#include <stdint.h>

#include "../../aerial_gym_simulator_b200/csrc/contact_core.cuh"

using namespace agx;

extern "C" {

// rows [total, stride] (read and written), mass [total], hull tables as AgxObstacleHull's with asset_file [total];
// kept [total, AGX_CONTACT_MAX] = the kept vertex indices deepest first (-1 = unused), count [total]
void shadow_obstacle_ground(long long total, const AgxContactParams* p, float* rows, int stride, const AgxObstacleMass* mass,
                            const float* vertices, const int32_t* file_offset, const float* file_reach, const int32_t* asset_file,
                            int32_t* kept, int32_t* count) {
    for (long long i = 0; i < total; ++i) {
        const int f = asset_file[i];
        const int v0 = file_offset[f];
        int k[AGX_CONTACT_MAX];
        const int n = obstacle_ground_row(*p, rows + i * stride, mass[i], vertices + (size_t)3 * v0, file_offset[f + 1] - v0,
                                          file_reach[f], k);
        for (int j = 0; j < AGX_CONTACT_MAX; ++j) kept[i * AGX_CONTACT_MAX + j] = j < n ? k[j] : -1;
        count[i] = n;
    }
}

}  // extern "C"
