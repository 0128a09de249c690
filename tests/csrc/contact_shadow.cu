// TEST INFRASTRUCTURE ONLY -- CPU shadow of the contact solves (aerial_gym_simulator_b200/csrc/contact_core.cuh).
//
// The code the contact kernels run after their contact search, compiled a second time as HOST code (-DAGX_HOST_SHADOW,
// -ffp-contract=off) and driven by a loop over envs or rows, so the CPU tests can hold the kernels' own arithmetic against
// oracle/contact*_oracle.py bit for bit on a machine without a GPU: the static solve of hp2_contact_kernel, the moving solve of
// hp2_contact_moving_kernel, the dynamic solve of hp2_contact_dynamic_kernel, obstacle_ground_contact_kernel's rows and
// obstacle_obstacle_contact_kernel's envs.  Nothing in the product loads this library.
#include <stdint.h>

#include <vector>

#include "../../aerial_gym_simulator_b200/csrc/contact_core.cuh"

using namespace agx;

namespace {
// contact i of env e from contacts [E, AGX_CONTACT_MAX, 7] = point xyz, normal xyz, depth
ContactPt contact_at(const float* contacts, int e, int i) {
    const float* s = contacts + ((size_t)e * AGX_CONTACT_MAX + i) * 7;
    return ContactPt{{s[0], s[1], s[2]}, {s[3], s[4], s[5]}, s[6]};
}
}  // namespace

extern "C" {

// contacts [E, AGX_CONTACT_MAX, 7]; count [E]
void shadow_contact_solve(int num_envs, const AgxContactParams* p, float* root_state, int stride, const float* contacts,
                          const int32_t* count, float* force, uint8_t* crashes) {
    for (int e = 0; e < num_envs; ++e) {
        ContactPt c[AGX_CONTACT_MAX];
        const int n = count[e];
        for (int i = 0; i < n; ++i) c[i] = contact_at(contacts, e, i);
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

// contacts [E, AGX_CONTACT_MAX, 7]; count [E]; u [E, AGX_CONTACT_MAX, 3] obstacle point velocities
void shadow_contact_solve_moving(int num_envs, const AgxContactParams* p, float* root_state, int stride, const float* contacts,
                                 const int32_t* count, const float* u, float* force, uint8_t* crashes) {
    for (int e = 0; e < num_envs; ++e) {
        ContactPt c[AGX_CONTACT_MAX];
        float ue[AGX_CONTACT_MAX][3];
        const int n = count[e];
        for (int i = 0; i < n; ++i) {
            c[i] = contact_at(contacts, e, i);
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

// contacts [E, AGX_CONTACT_MAX, 7]; count [E]; ids [E, AGX_CONTACT_MAX] (object index, K = ground);
// asset_state [E, A, stride] (read and written), obj_asset [E, K], mass [E, A]
void shadow_contact_solve_dynamic(int num_envs, const AgxContactParams* p, float* root_state, int stride, const float* contacts,
                                  const int32_t* count, const int32_t* ids, int K, float* asset_state, int A, int asset_stride,
                                  const int32_t* obj_asset, const AgxObstacleMass* mass, float* force, uint8_t* crashes) {
    for (int e = 0; e < num_envs; ++e) {
        ContactPt c[AGX_CONTACT_MAX];
        int id[AGX_CONTACT_MAX];
        const int n = count[e];
        for (int i = 0; i < n; ++i) {
            c[i] = contact_at(contacts, e, i);
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

// One env at a time in the order obstacle_obstacle_contact_kernel runs it: obstacle_box_world, then the pairs (i, j), i < j, in
// order through obstacle_box_near / obstacle_box_pair, appended until a pair no longer fits, then obstacle_contacts_solve and
// contact_body_store.  rows [E*A, stride] (read and written), mass [E*A], boxes [F,15], asset_file [E*A]; count [E] = the env's
// contact-list length, contacts [E, AGX_OBSTACLE_MAX_CONTACTS, 9] = p (3), n (3), depth, i, j of each listed contact (unused entries
// untouched)
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
