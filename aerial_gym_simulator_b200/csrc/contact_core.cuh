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

// ---- Obstacle-obstacle contact of free obstacles (agx_obstacle_obstacle_contact; DESIGN.md "Contact between free obstacles").
// Every asset is one oriented box.  box [15] (asset frame, AgxObstacleBoxes): centre, the three unit axes, the half extents.

// an asset's box in the world: centre c, axes a[3k..3k+2] (axis k), half extents h, bounding-sphere radius r = |h|
struct ObstacleBox {
    float c[3], a[9], h[3], r;
};

AGX_DEV void obstacle_box_world(const float* row, const float* box, ObstacleBox& b) {
    float R[9], t[3];
    cquat_R(row + 3, R);
    cmatvec(R, box, t);
    for (int k = 0; k < 3; ++k) b.c[k] = row[k] + t[k];
    for (int k = 0; k < 3; ++k) cmatvec(R, box + 3 + 3 * k, b.a + 3 * k);
    for (int k = 0; k < 3; ++k) b.h[k] = box[12 + k];
    b.r = sqrtf(cdot(b.h, b.h));
}

// broad phase: the bounding spheres are within contact_offset of each other
AGX_DEV bool obstacle_box_near(const AgxContactParams& P, const ObstacleBox& A, const ObstacleBox& B) {
    float d[3];
    for (int k = 0; k < 3; ++k) d[k] = B.c[k] - A.c[k];
    const float s = A.r + B.r + P.contact_offset;
    return cdot(d, d) <= s * s;
}

// separation of the two boxes along the unit axis L (d = B.c - A.c): |d.L| - (sum_k hA_k |a_k.L| + sum_k hB_k |b_k.L|)
AGX_DEV float obb_sep(const ObstacleBox& A, const ObstacleBox& B, const float* d, const float* L) {
    float rA = 0.0f, rB = 0.0f;
    for (int k = 0; k < 3; ++k) {
        rA = rA + A.h[k] * fabsf(cdot(A.a + 3 * k, L));
        rB = rB + B.h[k] * fabsf(cdot(B.a + 3 * k, L));
    }
    return fabsf(cdot(d, L)) - (rA + rB);
}

// Narrow phase of one pair: the separating-axis test on the 15 axes (faces of A, faces of B, a_i x b_j with i outer), and the
// contact manifold.  A pair with any axis separated by more than contact_offset has no contact.  Axis choice, largest separation
// (least penetration) with a bias, first in axis order on ties: B's face only if it beats A's by more than AGX_OBB_AXIS_TOL, an edge
// pair only if it beats both faces by more than AGX_OBB_AXIS_TOL; edge axes with |a_i x b_j|^2 < 1e-6 (near-parallel edges) are
// skipped.  Normal n: the chosen axis, pointing from A to B.
// Face axis: the incident face (of the other box, the one most anti-parallel to the reference face's outward normal, first axis on
// ties) is clipped against the reference face's four side planes; every clipped point whose separation s along the outward normal
// is <= contact_offset is a contact at the incident point moved s / 2 towards the reference face, depth -s.  Edge axis: one contact
// at the midpoint of the closest points of the two edges (each clamped to its edge), depth = -separation.  At most AGX_CONTACT_MAX
// (= 8, the most a clipped quad can have) are kept, ordered by contact_insert on the key s: deepest first, ties to the lower index
// in the clipped polygon.  c [AGX_CONTACT_MAX] gets them (normal from A to B); returns their number.
#define AGX_OBB_AXIS_TOL 1e-4f
AGX_DEV int obstacle_box_pair(const AgxContactParams& P, const ObstacleBox& A, const ObstacleBox& B, ContactPt* c) {
    float d[3];
    for (int k = 0; k < 3; ++k) d[k] = B.c[k] - A.c[k];
    const float co = P.contact_offset;
    float sA = 0.0f, sB = 0.0f, sE = 0.0f;
    int kA = 0, kB = 0, kE = -1;
    for (int k = 0; k < 3; ++k) {
        const float s = obb_sep(A, B, d, A.a + 3 * k);
        if (s > co) return 0;
        if (k == 0 || s > sA) {
            sA = s;
            kA = k;
        }
    }
    for (int k = 0; k < 3; ++k) {
        const float s = obb_sep(A, B, d, B.a + 3 * k);
        if (s > co) return 0;
        if (k == 0 || s > sB) {
            sB = s;
            kB = k;
        }
    }
    float LE[3] = {0.0f, 0.0f, 0.0f};
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            float L[3];
            ccross(A.a + 3 * i, B.a + 3 * j, L);
            const float l2 = cdot(L, L);
            if (l2 < 1e-6f) continue;
            const float inv = 1.0f / sqrtf(l2);
            for (int k = 0; k < 3; ++k) L[k] = L[k] * inv;
            const float s = obb_sep(A, B, d, L);
            if (s > co) return 0;
            if (kE < 0 || s > sE) {
                sE = s;
                kE = 3 * i + j;
                for (int k = 0; k < 3; ++k) LE[k] = L[k];
            }
        }
    const bool refB = sB > sA + AGX_OBB_AXIS_TOL;
    const float sF = refB ? sB : sA;
    float n[3];
    if (kE >= 0 && sE > sF + AGX_OBB_AXIS_TOL) {
        // edge a_i against edge b_j
        const int i = kE / 3, j = kE % 3;
        const float sg = cdot(d, LE) >= 0.0f ? 1.0f : -1.0f;
        for (int k = 0; k < 3; ++k) n[k] = LE[k] * sg;
        float pa[3], pb[3];
        for (int k = 0; k < 3; ++k) {
            pa[k] = A.c[k];
            pb[k] = B.c[k];
        }
        for (int m = 0; m < 3; ++m) {
            if (m != i) {
                const float s = cdot(A.a + 3 * m, n) >= 0.0f ? A.h[m] : -A.h[m];
                for (int k = 0; k < 3; ++k) pa[k] = pa[k] + A.a[3 * m + k] * s;
            }
            if (m != j) {
                const float s = cdot(B.a + 3 * m, n) > 0.0f ? -B.h[m] : B.h[m];
                for (int k = 0; k < 3; ++k) pb[k] = pb[k] + B.a[3 * m + k] * s;
            }
        }
        const float* da = A.a + 3 * i;
        const float* db = B.a + 3 * j;
        float w[3];
        for (int k = 0; k < 3; ++k) w[k] = pa[k] - pb[k];
        const float b = cdot(da, db), dd = cdot(da, w), e = cdot(db, w);
        const float den = 1.0f - b * b;
        const float ta = fminf(fmaxf((b * e - dd) / den, -A.h[i]), A.h[i]);
        const float tb = fminf(fmaxf((e - b * dd) / den, -B.h[j]), B.h[j]);
        for (int k = 0; k < 3; ++k) c[0].p[k] = ((pa[k] + da[k] * ta) + (pb[k] + db[k] * tb)) * 0.5f;
        for (int k = 0; k < 3; ++k) c[0].n[k] = n[k];
        c[0].depth = -sE;
        return 1;
    }
    // face: reference box R (face axis kr, outward normal nr towards the other box), incident box I
    const ObstacleBox& R = refB ? B : A;
    const ObstacleBox& I = refB ? A : B;
    const int kr = refB ? kB : kA;
    {
        const float sg = cdot(d, R.a + 3 * kr) >= 0.0f ? 1.0f : -1.0f;
        for (int k = 0; k < 3; ++k) n[k] = R.a[3 * kr + k] * sg;  // from A to B
    }
    float nr[3], fc[3];
    for (int k = 0; k < 3; ++k) nr[k] = refB ? -n[k] : n[k];
    for (int k = 0; k < 3; ++k) fc[k] = R.c[k] + nr[k] * R.h[kr];
    const int r1 = (kr + 1) % 3, r2 = (kr + 2) % 3;
    const float* t1 = R.a + 3 * r1;
    const float* t2 = R.a + 3 * r2;
    const float e1 = R.h[r1], e2 = R.h[r2];
    int m = 0;
    float best = fabsf(cdot(nr, I.a));
    for (int k = 1; k < 3; ++k) {
        const float v = fabsf(cdot(nr, I.a + 3 * k));
        if (v > best) {
            best = v;
            m = k;
        }
    }
    const float so = cdot(nr, I.a + 3 * m) > 0.0f ? -I.h[m] : I.h[m];
    const int u = (m + 1) % 3, v = (m + 2) % 3;
    // the incident face's corners in the reference frame (x along t1, y along t2, s along nr from the reference face)
    float poly[2][AGX_CONTACT_MAX][3];
    int np = 4;
    const float su[4] = {1.0f, -1.0f, -1.0f, 1.0f}, sv[4] = {1.0f, 1.0f, -1.0f, -1.0f};
    for (int q = 0; q < 4; ++q) {
        float rel[3];
        for (int k = 0; k < 3; ++k)
            rel[k] = ((I.c[k] + I.a[3 * m + k] * so) + I.a[3 * u + k] * (su[q] * I.h[u]) + I.a[3 * v + k] * (sv[q] * I.h[v])) - fc[k];
        poly[0][q][0] = cdot(rel, t1);
        poly[0][q][1] = cdot(rel, t2);
        poly[0][q][2] = cdot(rel, nr);
    }
    // Sutherland-Hodgman against x <= e1, -x <= e1, y <= e2, -y <= e2
    int cur = 0;
    for (int pl = 0; pl < 4 && np > 0; ++pl) {
        const int ax = pl >> 1;
        const float sg = (pl & 1) ? -1.0f : 1.0f, lim = ax ? e2 : e1;
        int no = 0;
        for (int q = 0; q < np; ++q) {
            const float* pc = poly[cur][q];
            const float* pp = poly[cur][q == 0 ? np - 1 : q - 1];
            const float dc = pc[ax] * sg - lim, dp = pp[ax] * sg - lim;
            if ((dc <= 0.0f) != (dp <= 0.0f)) {
                const float t = dp / (dp - dc);
                for (int k = 0; k < 3; ++k) poly[1 - cur][no][k] = pp[k] + (pc[k] - pp[k]) * t;
                ++no;
            }
            if (dc <= 0.0f) {
                for (int k = 0; k < 3; ++k) poly[1 - cur][no][k] = pc[k];
                ++no;
            }
        }
        np = no;
        cur = 1 - cur;
    }
    float key[AGX_CONTACT_MAX];
    int id[AGX_CONTACT_MAX];
    int nc = 0;
    for (int q = 0; q < np; ++q) {
        const float* pq = poly[cur][q];
        if (pq[2] > co) continue;
        ContactPt pt;
        const float hs = pq[2] * 0.5f;
        for (int k = 0; k < 3; ++k) {
            pt.p[k] = fc[k] + t1[k] * pq[0] + t2[k] * pq[1] + nr[k] * hs;
            pt.n[k] = n[k];
        }
        pt.depth = -pq[2];
        nc = contact_insert(c, key, id, nc, pt, pq[2], q);
    }
    return nc;
}

// one contact of the env's list: the pair's bodies (i < j), and the solve's per-contact state
struct ObstacleContact {
    ContactPt c;   // normal from body i to body j
    int i, j;
    float kn, bias, ln, lt[3];
};

// Sequential impulses over the env's contact list in order, `iterations` passes: obstacle_ground_row's per-contact step with body j
// in the place of the body and body i in the place of the ground.  Relative velocity u_j(p) - u_i(p), u = v + w x (p - x); inverse
// effective mass along d: the sum of both bodies' 1/m + (s x d) . I_w^-1 (s x d), s = p - c; impulse +dP to j, -dP to i.  A
// kinematic body (not free) is read and never changed.  Every body of the list needs to be loaded in B.
AGX_DEV void obstacle_contacts_solve(const AgxContactParams& P, ContactBody* B, ObstacleContact* L, int n) {
    for (int q = 0; q < n; ++q) {
        ObstacleContact& o = L[q];
        const ContactBody& bi = B[o.i];
        const ContactBody& bj = B[o.j];
        float si[3], sj[3];
        for (int k = 0; k < 3; ++k) {
            si[k] = o.c.p[k] - bi.c[k];
            sj[k] = o.c.p[k] - bj.c[k];
            o.lt[k] = 0.0f;
        }
        o.kn = ckeff(sj, o.c.n, bj.inv_m, bj.Iw) + ckeff(si, o.c.n, bi.inv_m, bi.Iw);
        o.bias = fminf(fmaxf(o.c.depth - P.rest_offset, 0.0f) / P.dt, P.max_depenetration_velocity);
        o.ln = 0.0f;
    }
    for (int it = 0; it < P.iterations; ++it) {
        for (int q = 0; q < n; ++q) {
            ObstacleContact& o = L[q];
            ContactBody& bi = B[o.i];
            ContactBody& bj = B[o.j];
            const float* nn = o.c.n;
            float ri[3], rj[3], si[3], sj[3];
            for (int k = 0; k < 3; ++k) {
                ri[k] = o.c.p[k] - bi.x[k];
                rj[k] = o.c.p[k] - bj.x[k];
                si[k] = o.c.p[k] - bi.c[k];
                sj[k] = o.c.p[k] - bj.c[k];
            }
            float vr[3], u[3], dP[3], nP[3];
            // normal: accumulated impulse >= 0, target separating velocity bias
            cvel(bj.v, bj.w, rj, vr);
            cvel(bi.v, bi.w, ri, u);
            for (int k = 0; k < 3; ++k) vr[k] = vr[k] - u[k];
            float dl = (o.bias - cdot(nn, vr)) / o.kn;
            const float l1 = fmaxf(o.ln + dl, 0.0f);
            dl = l1 - o.ln;
            o.ln = l1;
            for (int k = 0; k < 3; ++k) {
                dP[k] = nn[k] * dl;
                nP[k] = -dP[k];
            }
            if (bj.free) cbody_apply(dP, sj, bj);
            if (bi.free) cbody_apply(nP, si, bi);
            // friction: drive the tangential relative velocity at p to 0, accumulated impulse inside the circle mu * ln
            cvel(bj.v, bj.w, rj, vr);
            cvel(bi.v, bi.w, ri, u);
            for (int k = 0; k < 3; ++k) vr[k] = vr[k] - u[k];
            const float vn = cdot(nn, vr);
            float vt[3], l2[3];
            for (int k = 0; k < 3; ++k) {
                vt[k] = vr[k] - nn[k] * vn;
                l2[k] = o.lt[k];
            }
            const float s = sqrtf(cdot(vt, vt));
            if (s > 0.0f) {
                float t[3];
                for (int k = 0; k < 3; ++k) t[k] = vt[k] / s;
                const float dt_ = s / (ckeff(sj, t, bj.inv_m, bj.Iw) + ckeff(si, t, bi.inv_m, bi.Iw));
                for (int k = 0; k < 3; ++k) l2[k] = l2[k] - t[k] * dt_;
            }
            const float mag = sqrtf(cdot(l2, l2)), lim = P.friction * o.ln;
            if (mag > lim) {
                const float f = lim / mag;
                for (int k = 0; k < 3; ++k) l2[k] = l2[k] * f;
            }
            for (int k = 0; k < 3; ++k) {
                dP[k] = l2[k] - o.lt[k];
                o.lt[k] = l2[k];
                nP[k] = -dP[k];
            }
            if (bj.free) cbody_apply(dP, sj, bj);
            if (bi.free) cbody_apply(nP, si, bi);
        }
    }
}

}  // namespace agx
