// Robot-environment contact (DESIGN.md "Contact mode"): the robot's collision sphere against the scene objects and the ground
// plane, one velocity-level sequential-impulse solve after each physics sub-step.  This header holds the solve: a contact list in,
// the velocity change and the total impulse out.  The contact search (BVH descent, closest point) is in hp2_raycast.cu.
// AGX_DEV: device-only in the product (hp2_raycast.cu, compiled with -fmad=false), host+device in the CPU shadow build
// (tests/csrc/contact_shadow.cu, -ffp-contract=off).  oracle/contact_oracle.py restates every line in numpy float32 in the same
// operation order, so the three agree bit for bit.
#pragma once
#include "../../include/aerial_gym_b200.h"
#include "agx_math.cuh"

namespace agx {

struct ContactPt {
    float p[3];   // contact point, world frame
    float n[3];   // unit normal, from the obstacle towards the sphere centre
    float depth;  // penetration: radius - distance (negative while the sphere is inside the contact offset only)
};

// keep the AGX_CONTACT_MAX nearest contacts, ordered by (distance, id); id = object index, the ground plane has the largest id
AGX_DEV int contact_insert(ContactPt* c, float* key, int* id, int n, const ContactPt& pt, float k, int obj) {
    int i = n < AGX_CONTACT_MAX ? n : AGX_CONTACT_MAX - 1;
    if (n == AGX_CONTACT_MAX && !(k < key[i] || (k == key[i] && obj < id[i]))) return n;
    while (i > 0 && (k < key[i - 1] || (k == key[i - 1] && obj < id[i - 1]))) {
        c[i] = c[i - 1];
        key[i] = key[i - 1];
        id[i] = id[i - 1];
        --i;
    }
    c[i] = pt;
    key[i] = k;
    id[i] = obj;
    return n < AGX_CONTACT_MAX ? n + 1 : n;
}

AGX_DEV float cdot(const float* a, const float* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
AGX_DEV void ccross(const float* a, const float* b, float* o) {
    o[0] = a[1] * b[2] - a[2] * b[1];
    o[1] = a[2] * b[0] - a[0] * b[2];
    o[2] = a[0] * b[1] - a[1] * b[0];
}
AGX_DEV void cmatvec(const float* M, const float* x, float* o) {
    for (int i = 0; i < 3; ++i) o[i] = M[3 * i] * x[0] + M[3 * i + 1] * x[1] + M[3 * i + 2] * x[2];
}
// impulse P at lever arm r: v += P / m, w += I_w^-1 (r x P)
AGX_DEV void capply(const float* P, const float* r, float inv_m, const float* Iw, float* v, float* w) {
    float rp[3], dw[3];
    ccross(r, P, rp);
    cmatvec(Iw, rp, dw);
    for (int i = 0; i < 3; ++i) {
        v[i] = v[i] + P[i] * inv_m;
        w[i] = w[i] + dw[i];
    }
}
// inverse effective mass of the body along direction d at lever arm r
AGX_DEV float ckeff(const float* r, const float* d, float inv_m, const float* Iw) {
    float rd[3], m[3];
    ccross(r, d, rd);
    cmatvec(Iw, rd, m);
    return inv_m + cdot(rd, m);
}
// contact point velocity v + w x r
AGX_DEV void cvel(const float* v, const float* w, const float* r, float* o) {
    float wr[3];
    ccross(w, r, wr);
    for (int i = 0; i < 3; ++i) o[i] = v[i] + wr[i];
}
// velocity of a moving obstacle at the contact point p: its asset row (x y z qx qy qz qw vx vy vz wx wy wz) gives v + w x (p - x)
AGX_DEV void obstacle_point_vel(const float* row, const float* p, float* u) {
    const float r[3] = {p[0] - row[0], p[1] - row[1], p[2] - row[2]};
    cvel(row + 7, row + 10, r, u);
}

// One env: n contacts of the sphere whose centre is pos and orientation q (x, y, z, w).  v, w: world linear / angular velocity,
// updated in place.  imp: sum of the accumulated contact impulses (world frame).
// MOVING (agx_hp2_contact_moving): u[i] is the velocity of contact i's obstacle at its contact point, and both rows act on the
// relative velocity v_robot(p) - u.  The obstacle is kinematic (infinite mass), so only the robot's velocity changes.  Without
// MOVING no u is read and the code is the static solve's.
template <bool MOVING = false>
AGX_DEV void contact_solve(const AgxContactParams& P, const float* pos, const float* q, float* v, float* w, const ContactPt* c, int n,
                           float* imp, const float (*u)[3] = nullptr) {
    const float x = q[0], y = q[1], z = q[2], qw = q[3];
    float R[9];
    R[0] = 1.0f - 2.0f * (y * y + z * z);
    R[1] = 2.0f * (x * y - z * qw);
    R[2] = 2.0f * (x * z + y * qw);
    R[3] = 2.0f * (x * y + z * qw);
    R[4] = 1.0f - 2.0f * (x * x + z * z);
    R[5] = 2.0f * (y * z - x * qw);
    R[6] = 2.0f * (x * z - y * qw);
    R[7] = 2.0f * (y * z + x * qw);
    R[8] = 1.0f - 2.0f * (x * x + y * y);
    float com[3], A[9], Iw[9];
    cmatvec(R, P.com, com);
    for (int i = 0; i < 3; ++i) com[i] = pos[i] + com[i];
    for (int i = 0; i < 3; ++i)  // A = R I^-1, Iw = A R^T
        for (int j = 0; j < 3; ++j) A[3 * i + j] = R[3 * i] * P.inertia_inv[j] + R[3 * i + 1] * P.inertia_inv[3 + j] + R[3 * i + 2] * P.inertia_inv[6 + j];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) Iw[3 * i + j] = A[3 * i] * R[3 * j] + A[3 * i + 1] * R[3 * j + 1] + A[3 * i + 2] * R[3 * j + 2];
    const float inv_m = 1.0f / P.mass;
    float r[AGX_CONTACT_MAX][3], kn[AGX_CONTACT_MAX], bias[AGX_CONTACT_MAX], ln[AGX_CONTACT_MAX], lt[AGX_CONTACT_MAX][3];
    for (int i = 0; i < n; ++i) {
        for (int k = 0; k < 3; ++k) {
            r[i][k] = c[i].p[k] - com[k];
            lt[i][k] = 0.0f;
        }
        kn[i] = ckeff(r[i], c[i].n, inv_m, Iw);
        bias[i] = fminf(fmaxf(c[i].depth - P.rest_offset, 0.0f) / P.dt, P.max_depenetration_velocity);
        ln[i] = 0.0f;
    }
    for (int it = 0; it < P.iterations; ++it) {
        for (int i = 0; i < n; ++i) {
            const float* nn = c[i].n;
            float vr[3], dP[3];
            // normal: accumulated impulse >= 0, target separating velocity bias
            cvel(v, w, r[i], vr);
            if (MOVING)
                for (int k = 0; k < 3; ++k) vr[k] = vr[k] - u[i][k];
            float dl = (bias[i] - cdot(nn, vr)) / kn[i];
            const float l1 = fmaxf(ln[i] + dl, 0.0f);
            dl = l1 - ln[i];
            ln[i] = l1;
            for (int k = 0; k < 3; ++k) dP[k] = nn[k] * dl;
            capply(dP, r[i], inv_m, Iw, v, w);
            // friction: drive the tangential velocity to 0, accumulated impulse inside the circle mu * ln
            cvel(v, w, r[i], vr);
            if (MOVING)
                for (int k = 0; k < 3; ++k) vr[k] = vr[k] - u[i][k];
            const float vn = cdot(nn, vr);
            float vt[3], l2[3];
            for (int k = 0; k < 3; ++k) {
                vt[k] = vr[k] - nn[k] * vn;
                l2[k] = lt[i][k];
            }
            const float s = sqrtf(cdot(vt, vt));
            if (s > 0.0f) {
                float t[3];
                for (int k = 0; k < 3; ++k) t[k] = vt[k] / s;
                const float dt_ = s / ckeff(r[i], t, inv_m, Iw);
                for (int k = 0; k < 3; ++k) l2[k] = l2[k] - t[k] * dt_;
            }
            const float mag = sqrtf(cdot(l2, l2)), lim = P.friction * ln[i];
            if (mag > lim) {
                const float f = lim / mag;
                for (int k = 0; k < 3; ++k) l2[k] = l2[k] * f;
            }
            for (int k = 0; k < 3; ++k) {
                dP[k] = l2[k] - lt[i][k];
                lt[i][k] = l2[k];
            }
            capply(dP, r[i], inv_m, Iw, v, w);
        }
    }
    imp[0] = imp[1] = imp[2] = 0.0f;
    for (int i = 0; i < n; ++i)
        for (int k = 0; k < 3; ++k) imp[k] = imp[k] + c[i].n[k] * ln[i] + lt[i][k];
}

// the per-env epilogue: solve, contact force = impulse / dt, crash flag when |F| exceeds the threshold (the reference's rule)
template <bool MOVING = false>
AGX_DEV void contact_env(const AgxContactParams& P, float* rs, const ContactPt* c, int n, float* force, uint8_t* crash,
                         const float (*u)[3] = nullptr) {
    float v[3] = {rs[7], rs[8], rs[9]}, w[3] = {rs[10], rs[11], rs[12]}, imp[3];
    contact_solve<MOVING>(P, rs, rs + 3, v, w, c, n, imp, u);
    for (int k = 0; k < 3; ++k) {
        rs[7 + k] = v[k];
        rs[10 + k] = w[k];
        force[k] = imp[k] / P.dt;
    }
    if (sqrtf(cdot(force, force)) > P.force_threshold) *crash = 1;
}

// ---- Dynamic obstacles (agx_hp2_contact_dynamic): each obstacle asset is a free rigid body of finite mass, and every contact
// impulse acts on the robot and on that body.  Separate functions, so that the static and moving instantiations above keep their
// machine code.

// One obstacle asset in the two-body solve.  Its twist is kept in the asset row's form: v is the velocity of the asset's origin x
// (not of its COM c), w the angular velocity, both world frame.
struct ContactBody {
    float x[3], q[4], v[3], w[3];  // the asset row: origin, orientation (x, y, z, w), twist (updated by the solve)
    float c[3];                    // COM, world
    float oc[3];                   // x - c
    float inv_m;
    float Iw[9];                   // world inverse inertia R I^-1 R^T
    bool free;                     // inv_m > 0 or a non-zero inverse inertia; otherwise kinematic: the solve reads its twist only
};

// R (row-major) of the unit quaternion q (x, y, z, w): contact_solve's expressions
AGX_DEV void cquat_R(const float* q, float* R) {
    const float x = q[0], y = q[1], z = q[2], qw = q[3];
    R[0] = 1.0f - 2.0f * (y * y + z * z);
    R[1] = 2.0f * (x * y - z * qw);
    R[2] = 2.0f * (x * z + y * qw);
    R[3] = 2.0f * (x * y + z * qw);
    R[4] = 1.0f - 2.0f * (x * x + z * z);
    R[5] = 2.0f * (y * z - x * qw);
    R[6] = 2.0f * (x * z - y * qw);
    R[7] = 2.0f * (y * z + x * qw);
    R[8] = 1.0f - 2.0f * (x * x + y * y);
}

// world inverse inertia R I^-1 R^T, in contact_solve's order (A = R I^-1, Iw = A R^T)
AGX_DEV void cworld_inv_inertia(const float* R, const float* ii, float* Iw) {
    float A[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) A[3 * i + j] = R[3 * i] * ii[j] + R[3 * i + 1] * ii[3 + j] + R[3 * i + 2] * ii[6 + j];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) Iw[3 * i + j] = A[3 * i] * R[3 * j] + A[3 * i + 1] * R[3 * j + 1] + A[3 * i + 2] * R[3 * j + 2];
}

// the body of an asset row (x y z qx qy qz qw vx vy vz wx wy wz) and its mass-table entry
AGX_DEV void contact_body_load(ContactBody& b, const float* row, const AgxObstacleMass& m) {
    for (int k = 0; k < 3; ++k) {
        b.x[k] = row[k];
        b.v[k] = row[7 + k];
        b.w[k] = row[10 + k];
    }
    for (int k = 0; k < 4; ++k) b.q[k] = row[3 + k];
    float R[9], cm[3];
    cquat_R(b.q, R);
    cmatvec(R, m.com, cm);
    for (int k = 0; k < 3; ++k) {
        b.c[k] = b.x[k] + cm[k];
        b.oc[k] = b.x[k] - b.c[k];
    }
    cworld_inv_inertia(R, m.inertia_inv, b.Iw);
    b.inv_m = m.inv_mass;
    bool rot = false;
    for (int k = 0; k < 9; ++k) rot = rot || m.inertia_inv[k] != 0.0f;
    b.free = m.inv_mass > 0.0f || rot;
}

// one env's bodies: the asset of each kept object contact (id < K; the ground has id K), one body per distinct asset in the order of
// its first contact.  obj_asset [K], asset rows [A, stride] and mass [A] of this env.  body[i] = contact i's body, -1 for the
// ground; rows[b] = body b's asset row.  Returns the number of bodies (<= n).
AGX_DEV int contact_bodies_gather(const int* id, int n, int K, const int32_t* obj_asset, float* asset_rows, int stride,
                                  const AgxObstacleMass* mass, ContactBody* B, float** rows, int* body) {
    int asset[AGX_CONTACT_MAX];
    int nb = 0;
    for (int i = 0; i < n; ++i) {
        body[i] = -1;
        if (id[i] >= K) continue;
        const int a = obj_asset[id[i]];
        int j = 0;
        while (j < nb && asset[j] != a) ++j;
        if (j == nb) {
            asset[nb] = a;
            rows[nb] = asset_rows + (size_t)a * stride;
            contact_body_load(B[nb], rows[nb], mass[a]);
            ++nb;
        }
        body[i] = j;
    }
    return nb;
}

// impulse P on the body at lever arm s from its COM: w += I_w^-1 (s x P), v (of the origin) += P / m + dw x (x - c)
AGX_DEV void cbody_apply(const float* P, const float* s, ContactBody& b) {
    float sp[3], dw[3], dwx[3];
    ccross(s, P, sp);
    cmatvec(b.Iw, sp, dw);
    ccross(dw, b.oc, dwx);
    for (int k = 0; k < 3; ++k) {
        b.w[k] = b.w[k] + dw[k];
        b.v[k] = b.v[k] + (P[k] * b.inv_m + dwx[k]);
    }
}

// contact_solve with two bodies per contact: body[i] is the index in B of contact i's obstacle, -1 for the ground (at rest,
// infinite mass).  The relative velocity is v_robot(p) - (v_a + w_a x (p - x_a)); the inverse effective mass along d adds the
// body's 1/m_a + (s x d) . I_a,w^-1 (s x d) with s = p - c_a; each impulse dP goes +dP to the robot and -dP to the body.  Contacts
// on one body see each other's updates within a pass.  With every body kinematic the arithmetic is contact_solve<true>'s.
AGX_DEV void contact_solve_dynamic(const AgxContactParams& P, const float* pos, const float* q, float* v, float* w, const ContactPt* c,
                                   int n, float* imp, const int* body, ContactBody* B) {
    float R[9], com[3], Iw[9];
    cquat_R(q, R);
    cmatvec(R, P.com, com);
    for (int i = 0; i < 3; ++i) com[i] = pos[i] + com[i];
    cworld_inv_inertia(R, P.inertia_inv, Iw);
    const float inv_m = 1.0f / P.mass;
    float r[AGX_CONTACT_MAX][3], ra[AGX_CONTACT_MAX][3], sa[AGX_CONTACT_MAX][3];
    float kn[AGX_CONTACT_MAX], bias[AGX_CONTACT_MAX], ln[AGX_CONTACT_MAX], lt[AGX_CONTACT_MAX][3];
    for (int i = 0; i < n; ++i) {
        const int b = body[i];
        for (int k = 0; k < 3; ++k) {
            r[i][k] = c[i].p[k] - com[k];
            ra[i][k] = b >= 0 ? c[i].p[k] - B[b].x[k] : 0.0f;
            sa[i][k] = b >= 0 ? c[i].p[k] - B[b].c[k] : 0.0f;
            lt[i][k] = 0.0f;
        }
        kn[i] = ckeff(r[i], c[i].n, inv_m, Iw);
        if (b >= 0) kn[i] = kn[i] + ckeff(sa[i], c[i].n, B[b].inv_m, B[b].Iw);
        bias[i] = fminf(fmaxf(c[i].depth - P.rest_offset, 0.0f) / P.dt, P.max_depenetration_velocity);
        ln[i] = 0.0f;
    }
    for (int it = 0; it < P.iterations; ++it) {
        for (int i = 0; i < n; ++i) {
            const float* nn = c[i].n;
            const int b = body[i];
            float vr[3], u[3], dP[3], nP[3];
            // normal: accumulated impulse >= 0, target separating velocity bias
            cvel(v, w, r[i], vr);
            if (b >= 0) {
                cvel(B[b].v, B[b].w, ra[i], u);
                for (int k = 0; k < 3; ++k) vr[k] = vr[k] - u[k];
            }
            float dl = (bias[i] - cdot(nn, vr)) / kn[i];
            const float l1 = fmaxf(ln[i] + dl, 0.0f);
            dl = l1 - ln[i];
            ln[i] = l1;
            for (int k = 0; k < 3; ++k) dP[k] = nn[k] * dl;
            capply(dP, r[i], inv_m, Iw, v, w);
            if (b >= 0 && B[b].free) {
                for (int k = 0; k < 3; ++k) nP[k] = -dP[k];
                cbody_apply(nP, sa[i], B[b]);
            }
            // friction: drive the tangential relative velocity to 0, accumulated impulse inside the circle mu * ln
            cvel(v, w, r[i], vr);
            if (b >= 0) {
                cvel(B[b].v, B[b].w, ra[i], u);
                for (int k = 0; k < 3; ++k) vr[k] = vr[k] - u[k];
            }
            const float vn = cdot(nn, vr);
            float vt[3], l2[3];
            for (int k = 0; k < 3; ++k) {
                vt[k] = vr[k] - nn[k] * vn;
                l2[k] = lt[i][k];
            }
            const float s = sqrtf(cdot(vt, vt));
            if (s > 0.0f) {
                float t[3];
                for (int k = 0; k < 3; ++k) t[k] = vt[k] / s;
                float kt = ckeff(r[i], t, inv_m, Iw);
                if (b >= 0) kt = kt + ckeff(sa[i], t, B[b].inv_m, B[b].Iw);
                const float dt_ = s / kt;
                for (int k = 0; k < 3; ++k) l2[k] = l2[k] - t[k] * dt_;
            }
            const float mag = sqrtf(cdot(l2, l2)), lim = P.friction * ln[i];
            if (mag > lim) {
                const float f = lim / mag;
                for (int k = 0; k < 3; ++k) l2[k] = l2[k] * f;
            }
            for (int k = 0; k < 3; ++k) {
                dP[k] = l2[k] - lt[i][k];
                lt[i][k] = l2[k];
            }
            capply(dP, r[i], inv_m, Iw, v, w);
            if (b >= 0 && B[b].free) {
                for (int k = 0; k < 3; ++k) nP[k] = -dP[k];
                cbody_apply(nP, sa[i], B[b]);
            }
        }
    }
    imp[0] = imp[1] = imp[2] = 0.0f;
    for (int i = 0; i < n; ++i)
        for (int k = 0; k < 3; ++k) imp[k] = imp[k] + c[i].n[k] * ln[i] + lt[i][k];
}

// write a free body back to its asset row: the new twist, and the first-order position correction x += dt dv,
// q = normalize(dq(dw dt) (x) q) with dq(a) = (a / 2, 1), dv / dw = the solve's change of the twist.  The rest of the sub-step
// then moves the obstacle with its post-solve velocity.
AGX_DEV void contact_body_store(const ContactBody& b, float* row, float dt) {
    float h[3];
    for (int k = 0; k < 3; ++k) {
        row[k] = b.x[k] + (b.v[k] - row[7 + k]) * dt;
        h[k] = (b.w[k] - row[10 + k]) * dt * 0.5f;
    }
    const float* q = b.q;  // (h, 1) (x) q, Hamilton product
    float qn[4];
    qn[0] = q[0] + h[0] * q[3] + h[1] * q[2] - h[2] * q[1];
    qn[1] = q[1] - h[0] * q[2] + h[1] * q[3] + h[2] * q[0];
    qn[2] = q[2] + h[0] * q[1] - h[1] * q[0] + h[2] * q[3];
    qn[3] = q[3] - h[0] * q[0] - h[1] * q[1] - h[2] * q[2];
    const float inv = 1.0f / sqrtf(qn[0] * qn[0] + qn[1] * qn[1] + qn[2] * qn[2] + qn[3] * qn[3]);
    for (int k = 0; k < 4; ++k) row[3 + k] = qn[k] * inv;
    for (int k = 0; k < 3; ++k) {
        row[7 + k] = b.v[k];
        row[10 + k] = b.w[k];
    }
}

// contact_env for dynamic obstacles: the two-body solve, the robot's outputs as contact_env writes them, then every free body of
// B[0..nb) written back to rows[b]
AGX_DEV void contact_env_dynamic(const AgxContactParams& P, float* rs, const ContactPt* c, int n, float* force, uint8_t* crash,
                                 const int* body, ContactBody* B, int nb, float* const* rows) {
    float v[3] = {rs[7], rs[8], rs[9]}, w[3] = {rs[10], rs[11], rs[12]}, imp[3];
    contact_solve_dynamic(P, rs, rs + 3, v, w, c, n, imp, body, B);
    for (int k = 0; k < 3; ++k) {
        rs[7 + k] = v[k];
        rs[10 + k] = w[k];
        force[k] = imp[k] / P.dt;
    }
    if (sqrtf(cdot(force, force)) > P.force_threshold) *crash = 1;
    for (int b = 0; b < nb; ++b)
        if (B[b].free) contact_body_store(B[b], rows[b], P.dt);
}

// ---- Ground contact of free obstacles (agx_obstacle_ground_contact): one asset row against the plane z = 0 through the nv vertices
// verts [nv,3] (asset frame) of its geometry, reach >= their largest distance from the asset origin.  Contacts: every vertex below
// contact_offset, normal +z, depth -z, the AGX_CONTACT_MAX deepest kept (contact_insert on the key z: ties to the lower vertex index).
// Solve: contact_solve_dynamic's per-contact step with the body alone against the ground at rest (infinite mass), then
// contact_body_store.  Rows without a kept contact and kinematic rows are not written.  kept (may be NULL): the kept vertex
// indices, deepest first.  Returns the number kept (0 for a row skipped by the reach test or kinematic).
AGX_DEV int obstacle_ground_row(const AgxContactParams& P, float* row, const AgxObstacleMass& m, const float* verts, int nv, float reach,
                                int* kept) {
    if (row[2] - reach > P.contact_offset) return 0;
    ContactBody B;
    contact_body_load(B, row, m);
    if (!B.free) return 0;
    float R[9];
    cquat_R(B.q, R);
    ContactPt c[AGX_CONTACT_MAX];
    float key[AGX_CONTACT_MAX];
    int id[AGX_CONTACT_MAX];
    int n = 0;
    for (int j = 0; j < nv; ++j) {
        float rv[3];
        cmatvec(R, verts + 3 * j, rv);
        const float z = B.x[2] + rv[2];
        if (!(z < P.contact_offset)) continue;
        const ContactPt pt{{B.x[0] + rv[0], B.x[1] + rv[1], z}, {0.0f, 0.0f, 1.0f}, -z};
        n = contact_insert(c, key, id, n, pt, z, j);
    }
    if (kept)
        for (int i = 0; i < n; ++i) kept[i] = id[i];
    if (n == 0) return 0;
    float ra[AGX_CONTACT_MAX][3], sa[AGX_CONTACT_MAX][3];
    float kn[AGX_CONTACT_MAX], bias[AGX_CONTACT_MAX], ln[AGX_CONTACT_MAX], lt[AGX_CONTACT_MAX][3];
    for (int i = 0; i < n; ++i) {
        for (int k = 0; k < 3; ++k) {
            ra[i][k] = c[i].p[k] - B.x[k];
            sa[i][k] = c[i].p[k] - B.c[k];
            lt[i][k] = 0.0f;
        }
        kn[i] = ckeff(sa[i], c[i].n, B.inv_m, B.Iw);
        bias[i] = fminf(fmaxf(c[i].depth - P.rest_offset, 0.0f) / P.dt, P.max_depenetration_velocity);
        ln[i] = 0.0f;
    }
    for (int it = 0; it < P.iterations; ++it) {
        for (int i = 0; i < n; ++i) {
            const float* nn = c[i].n;
            float vr[3], dP[3];
            // normal: accumulated impulse >= 0, target separating velocity bias
            cvel(B.v, B.w, ra[i], vr);
            float dl = (bias[i] - cdot(nn, vr)) / kn[i];
            const float l1 = fmaxf(ln[i] + dl, 0.0f);
            dl = l1 - ln[i];
            ln[i] = l1;
            for (int k = 0; k < 3; ++k) dP[k] = nn[k] * dl;
            cbody_apply(dP, sa[i], B);
            // friction: drive the tangential velocity at p to 0, accumulated impulse inside the circle mu * ln
            cvel(B.v, B.w, ra[i], vr);
            const float vn = cdot(nn, vr);
            float vt[3], l2[3];
            for (int k = 0; k < 3; ++k) {
                vt[k] = vr[k] - nn[k] * vn;
                l2[k] = lt[i][k];
            }
            const float s = sqrtf(cdot(vt, vt));
            if (s > 0.0f) {
                float t[3];
                for (int k = 0; k < 3; ++k) t[k] = vt[k] / s;
                const float dt_ = s / ckeff(sa[i], t, B.inv_m, B.Iw);
                for (int k = 0; k < 3; ++k) l2[k] = l2[k] - t[k] * dt_;
            }
            const float mag = sqrtf(cdot(l2, l2)), lim = P.friction * ln[i];
            if (mag > lim) {
                const float f = lim / mag;
                for (int k = 0; k < 3; ++k) l2[k] = l2[k] * f;
            }
            for (int k = 0; k < 3; ++k) {
                dP[k] = l2[k] - lt[i][k];
                lt[i][k] = l2[k];
            }
            cbody_apply(dP, sa[i], B);
        }
    }
    contact_body_store(B, row, P.dt);
    return n;
}

}  // namespace agx
