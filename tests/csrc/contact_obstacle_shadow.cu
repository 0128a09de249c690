// TEST INFRASTRUCTURE ONLY -- CPU shadow of the obstacle-obstacle contact (aerial_gym_simulator_b200/csrc/contact_core.cuh,
// obstacle_box_world / obstacle_box_near / obstacle_box_pair / obstacle_contacts_solve / contact_body_store, in the order
// obstacle_obstacle_contact_kernel runs them for one env: the pairs (i, j), i < j, in order, appended until a pair no longer fits).
//
// Compiled as HOST code (-DAGX_HOST_SHADOW, -ffp-contract=off) like tests/csrc/contact_ground_shadow.cu, so
// tests/test_contact_obstacle_cpu.py can hold the kernel's own arithmetic against oracle/contact_obstacle_oracle.py bit for bit
// without a GPU.  Nothing in the product loads this library.
#include <stdint.h>

#include <vector>

#include "../../aerial_gym_simulator_b200/csrc/contact_core.cuh"

using namespace agx;

extern "C" {

// rows [E*A, stride] (read and written), mass [E*A], boxes [F,15], asset_file [E*A]; count [E] = the env's contact-list length,
// contacts [E, AGX_OBSTACLE_MAX_CONTACTS, 9] = p (3), n (3), depth, i, j of each listed contact (unused entries untouched)
void shadow_obstacle_obstacle(int E, int A, const AgxContactParams* p, float* rows, int stride, const AgxObstacleMass* mass,
                              const float* boxes, const int32_t* asset_file, int32_t* count, float* contacts) {
    std::vector<ContactBody> B(A);
    std::vector<ObstacleBox> X(A);
    std::vector<ObstacleContact> L(AGX_OBSTACLE_MAX_CONTACTS);
    for (int e = 0; e < E; ++e) {
        float* r = rows + (size_t)e * A * stride;
        for (int a = 0; a < A; ++a) {
            contact_body_load(B[a], r + (size_t)a * stride, mass[(size_t)e * A + a]);
            obstacle_box_world(r + (size_t)a * stride, boxes + (size_t)15 * asset_file[(size_t)e * A + a], X[a]);
        }
        int n = 0;
        bool full = false;
        for (int i = 0; i < A && !full; ++i)
            for (int j = i + 1; j < A; ++j) {
                if (!(B[i].free || B[j].free) || !obstacle_box_near(*p, X[i], X[j])) continue;
                ContactPt c[AGX_CONTACT_MAX];
                const int m = obstacle_box_pair(*p, X[i], X[j], c);
                if (m == 0) continue;
                if (n + m > AGX_OBSTACLE_MAX_CONTACTS) {
                    full = true;
                    break;
                }
                for (int k = 0; k < m; ++k) {
                    L[n + k].c = c[k];
                    L[n + k].i = i;
                    L[n + k].j = j;
                }
                n += m;
            }
        count[e] = n;
        for (int q = 0; q < n; ++q) {
            float* o = contacts + ((size_t)e * AGX_OBSTACLE_MAX_CONTACTS + q) * 9;
            for (int k = 0; k < 3; ++k) {
                o[k] = L[q].c.p[k];
                o[3 + k] = L[q].c.n[k];
            }
            o[6] = L[q].c.depth;
            o[7] = (float)L[q].i;
            o[8] = (float)L[q].j;
        }
        if (n == 0) continue;
        obstacle_contacts_solve(*p, B.data(), L.data(), n);
        std::vector<char> touched(A, 0);
        for (int q = 0; q < n; ++q) touched[L[q].i] = touched[L[q].j] = 1;
        for (int a = 0; a < A; ++a)
            if (touched[a] && B[a].free) contact_body_store(B[a], r + (size_t)a * stride, p->dt);
    }
}

}  // extern "C"
