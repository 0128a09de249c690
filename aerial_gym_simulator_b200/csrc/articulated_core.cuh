// Per-env arithmetic of the articulated-multirotor step (DESIGN.md "Articulated robots"): forward kinematics of the merged body
// tree, Featherstone's floating-base articulated-body algorithm (ABA) with the implicit joint drive, and the integration of base and
// joints.  The controller, allocation and motor model are hp1_core.cuh's, included and called unchanged.  Like hp1_core.cuh the
// text is compiled twice: device-only in libaerial_gym_b200.so (articulated.cu) and as host code in the CPU shadow of the test suite
// (tests/csrc/articulated_shadow.cu, -DAGX_HOST_SHADOW).
//
// Coordinates.  Every spatial quantity is expressed in ONE frame for all bodies: world axes, reference point O = the base origin at
// the start of the sub-step.  Plücker order (angular; linear): a motion vector is (w, v_O), the velocity of the body point that
// coincides with O; a force is (n_O, f).  With one common frame the ABA needs no spatial transforms between bodies (Featherstone,
// "Rigid Body Dynamics Algorithms", 2008, section 7.3 with every X the identity), and the lever arms stay of the size of the robot
// (~0.1 m), not of its distance from the world origin -- what keeps float32 usable.
#pragma once
#include <type_traits>

#include "../../include/aerial_gym_b200.h"
#include "agx_math.cuh"
#include "disturbance_core.cuh"
#include "hp1_core.cuh"

namespace agx {

// The instantiations of every articulated kernel, for its launcher in articulated.cu and for the CPU shadow alike: f(M, NB) with
// std::integral_constant arguments, M = 4 or 8 motors and the per-body scratch sized for the tree -- up to 9 bodies (a quadrotor
// with two joints per arm) or the full AGX_ART_MAX_BODIES.  Host code.
template <class F>
auto art_instantiation(int M, int B, F&& f) {
    using M4 = std::integral_constant<int, 4>;
    using M8 = std::integral_constant<int, 8>;
    using NB9 = std::integral_constant<int, 9>;
    using NBMax = std::integral_constant<int, AGX_ART_MAX_BODIES>;
    const bool small = B <= 9;
    if (M == 4) return small ? f(M4{}, NB9{}) : f(M4{}, NBMax{});
    return small ? f(M8{}, NB9{}) : f(M8{}, NBMax{});
}

AGX_DEV M33 ld33(const float* a) {
    M33 r;
#pragma unroll
    for (int i = 0; i < 9; ++i) r.m[i] = a[i];
    return r;
}
AGX_DEV M33 mul33(const M33& A, const M33& B) {
    M33 r;
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) r.m[3 * i + j] = A.m[3 * i] * B.m[j] + A.m[3 * i + 1] * B.m[3 + j] + A.m[3 * i + 2] * B.m[6 + j];
    return r;
}
AGX_DEV V3 mul33v(const M33& A, V3 v) {
    return V3{A.m[0] * v.x + A.m[1] * v.y + A.m[2] * v.z, A.m[3] * v.x + A.m[4] * v.y + A.m[5] * v.z,
              A.m[6] * v.x + A.m[7] * v.y + A.m[8] * v.z};
}
// rotation by angle t about the unit axis a (Rodrigues)
AGX_DEV M33 axis_angle(V3 a, float t) {
    float st, ct;
    sincos_(t, &st, &ct);
    const float k = 1.0f - ct;
    M33 r;
    r.m[0] = ct + k * a.x * a.x;       r.m[1] = k * a.x * a.y - st * a.z; r.m[2] = k * a.x * a.z + st * a.y;
    r.m[3] = k * a.y * a.x + st * a.z; r.m[4] = ct + k * a.y * a.y;       r.m[5] = k * a.y * a.z - st * a.x;
    r.m[6] = k * a.z * a.x - st * a.y; r.m[7] = k * a.z * a.y + st * a.x; r.m[8] = ct + k * a.z * a.z;
    return r;
}

AGX_DEV V3 sv_ang(const float* s) { return V3{s[0], s[1], s[2]}; }
AGX_DEV V3 sv_lin(const float* s) { return V3{s[3], s[4], s[5]}; }
AGX_DEV void sv_set(float* s, V3 a, V3 l) { s[0] = a.x; s[1] = a.y; s[2] = a.z; s[3] = l.x; s[4] = l.y; s[5] = l.z; }
AGX_DEV float sv_dot(const float* a, const float* b) {
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2] + a[3] * b[3] + a[4] * b[4] + a[5] * b[5];
}
// motion cross product v x u = (w x uw, w x ul + vl x uw)
AGX_DEV void crm(const float* v, const float* u, float* out) {
    const V3 w = sv_ang(v), vl = sv_lin(v), uw = sv_ang(u), ul = sv_lin(u);
    sv_set(out, cross(w, uw), cross(w, ul) + cross(vl, uw));
}
// force cross product v x* f = (w x n + vl x f, w x f)
AGX_DEV void crf(const float* v, const float* f, float* out) {
    const V3 w = sv_ang(v), vl = sv_lin(v), n = sv_ang(f), fl = sv_lin(f);
    sv_set(out, cross(w, n) + cross(vl, fl), cross(w, fl));
}
AGX_DEV void mul66(const float* I, const float* v, float* out) {
#pragma unroll
    for (int r = 0; r < 6; ++r) out[r] = I[6 * r] * v[0] + I[6 * r + 1] * v[1] + I[6 * r + 2] * v[2] + I[6 * r + 3] * v[3] +
                                         I[6 * r + 4] * v[4] + I[6 * r + 5] * v[5];
}
// rigid-body spatial inertia at O: mass m, COM c (relative to O), rotational inertia Ic about the COM (world axes)
//   [[Ic + m (c.c 1 - c c^T), m [c]x], [-m [c]x, m 1]]
AGX_DEV void rb_inertia(float m, V3 c, const M33& Ic, float* I) {
    const float cc = dot(c, c);
    const float cv[3] = {c.x, c.y, c.z};
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            I[6 * i + j] = Ic.m[3 * i + j] + m * ((i == j ? cc : 0.0f) - cv[i] * cv[j]);
            I[6 * (i + 3) + j + 3] = (i == j) ? m : 0.0f;
        }
    // m [c]x = m [[0,-cz,cy],[cz,0,-cx],[-cy,cx,0]]
    const float X[9] = {0.0f, -c.z, c.y, c.z, 0.0f, -c.x, -c.y, c.x, 0.0f};
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            I[6 * i + j + 3] = m * X[3 * i + j];
            I[6 * (i + 3) + j] = -m * X[3 * i + j];
        }
}
// solve A x = b for a symmetric positive definite 6x6 A (Cholesky, A not modified)
AGX_DEV void spd6_solve(const float* A, const float* b, float* x) {
    float L[21];  // lower triangle, row-major packed: L[i(i+1)/2 + j]
#pragma unroll
    for (int i = 0; i < 6; ++i)
#pragma unroll
        for (int j = 0; j <= i; ++j) {
            float s = A[6 * i + j];
#pragma unroll
            for (int k = 0; k < j; ++k) s -= L[i * (i + 1) / 2 + k] * L[j * (j + 1) / 2 + k];
            if (i == j) L[i * (i + 1) / 2 + i] = sqrtf(fmaxf(s, 1e-30f));
            else L[i * (i + 1) / 2 + j] = s / L[j * (j + 1) / 2 + j];
        }
    float y[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) {
        float s = b[i];
#pragma unroll
        for (int k = 0; k < i; ++k) s -= L[i * (i + 1) / 2 + k] * y[k];
        y[i] = s / L[i * (i + 1) / 2 + i];
    }
#pragma unroll
    for (int i = 5; i >= 0; --i) {
        float s = y[i];
#pragma unroll
        for (int k = i + 1; k < 6; ++k) s -= L[k * (k + 1) / 2 + i] * x[k];
        x[i] = s / L[i * (i + 1) / 2 + i];
    }
}

// R^T v
AGX_DEV V3 mul33tv(const M33& A, V3 v) {
    return V3{A.m[0] * v.x + A.m[3] * v.y + A.m[6] * v.z, A.m[1] * v.x + A.m[4] * v.y + A.m[7] * v.z,
              A.m[2] * v.x + A.m[5] * v.y + A.m[8] * v.z};
}

// ---- the IMU input of one body (agx_hp1_articulated_step_imu) ---------------------------------------------------------------
// From what the ABA holds for body b at the sub-step's start: its rotation R and origin P (relative to O), its spatial velocity
// V = (w, v_O) and acceleration A = (alpha, a^), both in world axes about O.  COM c = P + R com_b, its classical acceleration
// a_c = a^ + alpha x c + w x (v_O + w x c).  out [9] = (f, n, w_b), all in body b's frame:
//   f = m_b R^T (a_c - g)                       the non-gravitational force on the body, joint reactions included
//   n = I_b R^T alpha + w_b x I_b w_b            the net torque about the COM (I_b about the COM, body axes)
//   w_b = R^T w
AGX_DEV void art_imu_input(const AgxArticulation& art, int b, const M33& R, V3 P, const float* V, const float* A, V3 grav, float* out) {
    const V3 w = sv_ang(V), al = sv_ang(A);
    const V3 c = P + mul33v(R, ld3(art.com[b]));
    const V3 ac = sv_lin(A) + cross(al, c) + cross(w, sv_lin(V) + cross(w, c));
    const V3 f = mul33tv(R, (ac - grav) * art.mass[b]);
    const V3 wb = mul33tv(R, w), ab = mul33tv(R, al);
    const M33 Ib = ld33(art.inertia[b]);
    const V3 n = mul33v(Ib, ab) + cross(wb, mul33v(Ib, wb));
    out[0] = f.x; out[1] = f.y; out[2] = f.z;
    out[3] = n.x; out[4] = n.y; out[5] = n.z;
    out[6] = wb.x; out[7] = wb.y; out[8] = wb.z;
}

// ---- the joint force of one body (agx_hp1_articulated_step_joint_force) ------------------------------------------------------
// After the ABA's backward pass, body i's articulated inertia I^A and bias force p^A are final (only its ancestors' are still summed
// into), and the forward pass gives its acceleration A; f = I^A A + p^A = (n_O; F) is the spatial force the parent exerts on the
// subtree of body i through joint i, world axes about O.  out [6] = (R^T F, R^T (n_O - P x F)): the force, then the torque about the
// joint origin P, both in body i's frame; *dof = axis_i . (that torque) = S_i^T f, the joint torque of the implicit drive at the
// unprojected end-of-step state (DESIGN.md "Joint force sensing").
AGX_DEV void art_joint_force(const AgxArticulation& art, int i, const M33& R, V3 P, const float* IA, const float* PA, const float* A,
                             float* out, float* dof) {
    float f[6];
    mul66(IA, A, f);
    const V3 Fw{f[3] + PA[3], f[4] + PA[4], f[5] + PA[5]};
    const V3 nw{f[0] + PA[0], f[1] + PA[1], f[2] + PA[2]};
    const V3 F = mul33tv(R, Fw), n = mul33tv(R, nw - cross(P, Fw));
    out[0] = F.x; out[1] = F.y; out[2] = F.z;
    out[3] = n.x; out[4] = n.y; out[5] = n.z;
    *dof = dot(ld3(art.axis[i]), n);
}

// w_b = R_b^T w_b of body b without the dynamics (the IMU input of a launch with physics_steps = 0): the forward kinematics of
// art_dynamics along the bodies 0..b.  PRISM: the joints of the bodies set in pmask are prismatic (art_dynamics' PRISM).
template <int NB, bool PRISM = false>
AGX_DEV V3 art_body_angvel(const AgxArticulation& art, const EnvState& s, const float* q, const float* qd, int b, uint32_t pmask = 0) {
    M33 R[NB];
    V3 W[NB];
    R[0] = quat_to_matrix(s.q);
    W[0] = s.w;
    for (int i = 1; i <= b; ++i) {
        const int l = art.parent[i];
        const V3 ax = ld3(art.axis[i]);
        const M33 RJ = mul33(R[l], ld33(art.joint_R[i]));
        if constexpr (PRISM) {
            if ((pmask >> i) & 1u) {  // a slider turns nothing
                R[i] = RJ;
                W[i] = W[l];
                continue;
            }
        }
        R[i] = mul33(RJ, axis_angle(ax, q[i - 1]));
        W[i] = W[l] + mul33v(RJ, ax) * qd[i - 1];
    }
    return mul33tv(R[b], W[b]);
}

// ---- the dynamics of one sub-step ------------------------------------------------------------------------------------------
// In: base pose / twist s (root-origin velocity v, world angular velocity w), joint q, qd and drive targets qs, qds, motor thrusts
// (M motors), the base's external force F_w / torque T_w (world frame, force acting at the base origin), gravity, dt.
// Out: a0 = the base's spatial acceleration at O (angular; linear -- the linear part is NOT the classical acceleration of the base
// origin: that is a0_lin + w x v), qdd[D].
// The joint drive tau = k (qs - q') + d (qds - qd') is taken at the end-of-step q' = q + dt qd', qd' = qd + dt qdd: its implicit part
// moves into the joint's pivot D_i = S^T I^A S + dt d + dt^2 k, the explicit part k (qs - q - dt qd) + d (qds - qd) into u_i.
// IMU: where imu != NULL, also art_imu_input of body imu_body into imu[9]; a0 and qdd are the same either way.
// EFFORT: the joints with eff->effort_dof[i] set are torque-driven: qs holds their tau_e and their k is 0, so the explicit force is
// tau_e - d qd (d = the URDF damping alone, passive) and the pivot S^T I^A S + dt d.
// JFORCE: where jw != NULL, also art_joint_force of every body i >= 1 into jw + 6 i and jdof + i - 1, and zeros into jw[0..5].
// PRISM: the joint of every body i set in pmask is prismatic, a translation by q along its axis a = R_l joint_R_i axis_i: R_i =
// R_l joint_R_i, P_i = P_l + R_l joint_p_i + a q and S_i = (0, a); its drive force is the same law in N, and its jdof entry is
// axis_i . (the force of its jw row).  The other joints are stepped as without it.
template <int NB, bool IMU = false, bool EFFORT = false, bool JFORCE = false, bool PRISM = false>
AGX_DEV void art_dynamics(const AgxArticulation& art, const EnvState& s, const float* q, const float* qd, const float* qs,
                          const float* qds, float dt, V3 grav, int M, const float* thrust, V3 F_w, V3 T_w, float* a0, float* qdd,
                          int imu_body = 0, float* imu = nullptr, const AgxJointEffort* eff = nullptr, float* jw = nullptr,
                          float* jdof = nullptr, uint32_t pmask = 0) {
    const int B = art.num_bodies;
    M33 R[NB];
    V3 P[NB];
    float S[NB][6], V[NB][6], Cb[NB][6], IA[NB][36], PA[NB][6], U[NB][6], Dinv[NB], uu[NB];
    // forward kinematics, velocities, velocity-product terms, rigid inertias and bias forces (gravity included)
    R[0] = quat_to_matrix(s.q);
    P[0] = V3{0.0f, 0.0f, 0.0f};
    sv_set(V[0], s.w, s.v);
    for (int i = 0; i < B; ++i) {
        if (i > 0) {
            const int l = art.parent[i];
            const V3 ax = ld3(art.axis[i]);
            const M33 RJ = mul33(R[l], ld33(art.joint_R[i]));
            bool slide = false;
            if constexpr (PRISM) slide = (pmask >> i) & 1u;
            if (slide) {
                const V3 aw = mul33v(RJ, ax);
                R[i] = RJ;
                P[i] = P[l] + mul33v(R[l], ld3(art.joint_p[i])) + aw * q[i - 1];
                sv_set(S[i], V3{0.0f, 0.0f, 0.0f}, aw);
            } else {
                R[i] = mul33(RJ, axis_angle(ax, q[i - 1]));
                P[i] = P[l] + mul33v(R[l], ld3(art.joint_p[i]));
                const V3 aw = mul33v(RJ, ax);  // = R[i] ax
                sv_set(S[i], aw, cross(P[i], aw));
            }
            float vj[6];
#pragma unroll
            for (int k = 0; k < 6; ++k) vj[k] = S[i][k] * qd[i - 1];
#pragma unroll
            for (int k = 0; k < 6; ++k) V[i][k] = V[l][k] + vj[k];
            crm(V[i], vj, Cb[i]);
        }
        const float m = art.mass[i];
        const V3 c = P[i] + mul33v(R[i], ld3(art.com[i]));
        const M33 Ib = ld33(art.inertia[i]);
        // R Ib R^T
        M33 RI = mul33(R[i], Ib), Ic;
#pragma unroll
        for (int a = 0; a < 3; ++a)
#pragma unroll
            for (int b = 0; b < 3; ++b)
                Ic.m[3 * a + b] = RI.m[3 * a] * R[i].m[3 * b] + RI.m[3 * a + 1] * R[i].m[3 * b + 1] + RI.m[3 * a + 2] * R[i].m[3 * b + 2];
        rb_inertia(m, c, Ic, IA[i]);
        float h[6];
        mul66(IA[i], V[i], h);
        crf(V[i], h, PA[i]);
        const V3 fg = grav * m;  // gravity at the COM
        const V3 ng = cross(c, fg);
        PA[i][0] -= ng.x; PA[i][1] -= ng.y; PA[i][2] -= ng.z;
        PA[i][3] -= fg.x; PA[i][4] -= fg.y; PA[i][5] -= fg.z;
    }
    // motors: thrust f z_m at the motor link origin, reaction torque motor_torque f z_m (LOCAL_SPACE application)
    for (int k = 0; k < M; ++k) {
        const int b = art.motor_body[k];
        const M33 Rm = mul33(R[b], ld33(art.motor_R[k]));
        const V3 ez{Rm.m[2], Rm.m[5], Rm.m[8]};
        const V3 pos = P[b] + mul33v(R[b], ld3(art.motor_p[k]));
        const V3 f = ez * thrust[k];
        const V3 n = cross(pos, f) + ez * (art.motor_torque[k] * thrust[k]);
        PA[b][0] -= n.x; PA[b][1] -= n.y; PA[b][2] -= n.z;
        PA[b][3] -= f.x; PA[b][4] -= f.y; PA[b][5] -= f.z;
    }
    // drag + disturbance on the base (force at O: no moment about O)
    PA[0][0] -= T_w.x; PA[0][1] -= T_w.y; PA[0][2] -= T_w.z;
    PA[0][3] -= F_w.x; PA[0][4] -= F_w.y; PA[0][5] -= F_w.z;
    // backward pass: articulated inertias and bias forces, children into parents
    for (int i = B - 1; i >= 1; --i) {
        const int l = art.parent[i];
        const int j = i - 1;
        const float k = art.stiffness[i], dd = art.damping[i];
        mul66(IA[i], S[i], U[i]);
        const float Dd = sv_dot(S[i], U[i]) + dt * dd + dt * dt * k;
        const float tau = (EFFORT && eff->effort_dof[i]) ? qs[j] - dd * qd[j] : k * (qs[j] - q[j] - dt * qd[j]) + dd * (qds[j] - qd[j]);
        const float u = tau - sv_dot(S[i], PA[i]);
        const float di = 1.0f / Dd;
        Dinv[i] = di;
        uu[i] = u;
        float Ia[36];
#pragma unroll
        for (int r = 0; r < 6; ++r)
#pragma unroll
            for (int cc = 0; cc < 6; ++cc) Ia[6 * r + cc] = IA[i][6 * r + cc] - U[i][r] * U[i][cc] * di;
        float t[6];
        mul66(Ia, Cb[i], t);
#pragma unroll
        for (int r = 0; r < 6; ++r) PA[l][r] += PA[i][r] + t[r] + U[i][r] * (u * di);
#pragma unroll
        for (int r = 0; r < 36; ++r) IA[l][r] += Ia[r];
    }
    // the floating base: I^A_0 a0 = -p^A_0
    float rhs[6];
#pragma unroll
    for (int r = 0; r < 6; ++r) rhs[r] = -PA[0][r];
    spd6_solve(IA[0], rhs, a0);
    // forward pass: joint accelerations
    float A[NB][6];
#pragma unroll
    for (int r = 0; r < 6; ++r) A[0][r] = a0[r];
    for (int i = 1; i < B; ++i) {
        const int l = art.parent[i];
        float ai[6];
#pragma unroll
        for (int r = 0; r < 6; ++r) ai[r] = A[l][r] + Cb[i][r];
        const float x = (uu[i] - sv_dot(U[i], ai)) * Dinv[i];
        qdd[i - 1] = x;
#pragma unroll
        for (int r = 0; r < 6; ++r) A[i][r] = ai[r] + S[i][r] * x;
        if constexpr (JFORCE) {
            if (jw) art_joint_force(art, i, R[i], P[i], IA[i], PA[i], A[i], jw + 6 * i, jdof + (i - 1));
            if constexpr (PRISM) {
                if (jw && ((pmask >> i) & 1u)) jdof[i - 1] = dot(ld3(art.axis[i]), ld3(jw + 6 * i));  // the force along the slide
            }
        }
    }
    if constexpr (JFORCE) {
        if (jw) {
#pragma unroll
            for (int r = 0; r < 6; ++r) jw[r] = 0.0f;
        }
    }
    if constexpr (IMU) {
        if (imu) art_imu_input(art, imu_body, R[imu_body], P[imu_body], V[imu_body], A[imu_body], grav, imu);
    }
}

// ---- integration: the base by the HP1 integrator spec (DESIGN.md section 3, integrate() of hp1_core.cuh) on the accelerations
// the ABA gives, the joints semi-implicitly, then the limit projection
AGX_DEV void art_integrate(const AgxHp1Config& cfg, const AgxArticulation& art, EnvState& s, const float* a0, float* q, float* qd,
                           const float* qdd) {
    const float dt = cfg.dt;
    // spatial -> classical: the acceleration of the base origin is a0_lin + w x v
    const V3 a = sv_lin(a0) + cross(s.w, s.v);
    V3 v = (s.v + a * dt) * fmaxf(0.0f, 1.0f - dt * cfg.linear_damping);
    float vn = norm3(v);
    if (vn > cfg.max_linear_velocity) v = v * (cfg.max_linear_velocity / vn);
    V3 W = quat_rotate_inverse(s.q, s.w);
    V3 al = quat_rotate_inverse(s.q, sv_ang(a0));
    V3 Wn = W + al * dt;
    V3 w = quat_rotate(s.q, Wn) * fmaxf(0.0f, 1.0f - dt * cfg.angular_damping);
    float wn = norm3(w);
    if (wn > cfg.max_angular_velocity) {
        w = w * (cfg.max_angular_velocity / wn);
        wn = norm3(w);
    }
    s.x = s.x + v * dt;
    float sh, ch;
    sincos_(0.5f * dt * wn, &sh, &ch);
    float so = (wn > 0.0f) ? sh / wn : 0.0f;
    Q4 dq{w.x * so, w.y * so, w.z * so, ch};
    Q4 qn = quat_mul(dq, s.q);
    float inv = 1.0f / sqrtf(qn.x * qn.x + qn.y * qn.y + qn.z * qn.z + qn.w * qn.w);
    s.q = Q4{qn.x * inv, qn.y * inv, qn.z * inv, qn.w * inv};
    s.v = v;
    s.w = w;
    for (int j = 0; j < art.num_dofs; ++j) {
        float v1 = qd[j] + dt * qdd[j];
        float q1 = q[j] + dt * v1;
        if (art.limited[j + 1]) {  // projection, not a constraint: clamp q, drop the velocity that points out of the range
            const float lo = art.lower[j + 1], hi = art.upper[j + 1];
            if (q1 <= lo) { q1 = lo; v1 = fmaxf(v1, 0.0f); }
            if (q1 >= hi) { q1 = hi; v1 = fminf(v1, 0.0f); }
        }
        q[j] = q1;
        qd[j] = v1;
    }
}

// per-env parameters (the same values hp1.cu's load_params reads: per-env array or the config constant)
template <int M>
AGX_DEV void art_load_params(const AgxHp1Config& cfg, const AgxHp1Buffers& buf, int env, EnvParams<M>& p) {
#pragma unroll
    for (int i = 0; i < M; ++i) {
        p.thrust[i] = buf.motor_thrust[(size_t)env * M + i];
        p.tau_inc[i] = buf.tau_inc ? buf.tau_inc[(size_t)env * M + i] : cfg.tau_inc;
        p.tau_dec[i] = buf.tau_dec ? buf.tau_dec[(size_t)env * M + i] : cfg.tau_dec;
        p.k[i] = buf.k_thrust ? buf.k_thrust[(size_t)env * M + i] : cfg.k_thrust;
    }
    p.g.kp = buf.K_pos ? ld3(buf.K_pos + (size_t)env * 3) : ld3c(cfg.K_pos);
    p.g.kv = buf.K_vel ? ld3(buf.K_vel + (size_t)env * 3) : ld3c(cfg.K_vel);
    p.g.kr = buf.K_rot ? ld3(buf.K_rot + (size_t)env * 3) : ld3c(cfg.K_rot);
    p.g.kw = buf.K_angvel ? ld3(buf.K_angvel + (size_t)env * 3) : ld3c(cfg.K_angvel);
}

// ---- one env over cfg.physics_steps sub-steps (the kernel's thread body and the shadow's loop body) -------------------------
// Each sub-step: update_states -> controller -> allocation -> motor model (hp1_core.cuh), drag on the base (body-frame velocities
// of the base origin, base_multirotor.py:260-285) plus the disturbance, then the articulated dynamics and the integration.
// Derived states d are those of the last sub-step's start (agx_hp1_physics_step's staleness).
// IMU: also the IMU input of body imu_body into imu_input [N,9] -- art_imu_input on the last sub-step; with physics_steps = 0,
// f = n = 0 and w_b of the unstepped state (agx_hp1_physics_step's body_wrench is zero then).  The state arithmetic is unchanged.
// EFFORT: the effort DOFs of eff take tau_e = their entry of eff->effort, clamped to +-effort_limit where that is > 0, read once and
// held in qs for every sub-step (art_dynamics' EFFORT); the other DOFs are stepped as without it.
// JFORCE (with IMU and EFFORT): also the joint forces of the last sub-step into THIS env's rows, joint_wrench [B,6] and
// dof_force [D] (art_dynamics' JFORCE; the kernel points them at shared memory), both zero with physics_steps = 0.  The IMU input is written only where imu_input != NULL, and an eff
// without effort DOFs steps every DOF as the plain step does.  The state arithmetic is unchanged.
// PRISM (with JFORCE): the joints of the bodies set in pmask are prismatic (art_dynamics' PRISM), and the joint forces are written
// only where joint_wrench != NULL.
template <int M, int NB, bool IMU = false, bool EFFORT = false, bool JFORCE = false, bool PRISM = false>
AGX_DEV void art_env_step(const AgxHp1Config& cfg, const AgxHp1Buffers& buf, const AgxArticulation& art, int env, int imu_body = 0,
                          float* imu_input = nullptr, const AgxJointEffort* eff = nullptr, float* joint_wrench = nullptr,
                          float* dof_force = nullptr, uint32_t pmask = 0) {
    EnvParams<M> p;
    art_load_params<M>(cfg, buf, env, p);
    const int A = cfg.num_actions;
    float act[AGX_MAX_MOTORS];
#pragma unroll
    for (int i = 0; i < AGX_MAX_MOTORS; ++i) act[i] = (i < A) ? buf.actions[(size_t)env * A + i] : 0.0f;
#pragma unroll
    for (int i = 0; i < AGX_MAX_MOTORS; ++i) act[i] = fminf(fmaxf(act[i], -10.0f), 10.0f);  // clip_actions
    EnvState s = unpack(buf.root_state + (size_t)env * 13);
    const int D = art.num_dofs;
    float q[NB], qd[NB], qs[NB], qds[NB], qdd[NB];
    for (int j = 0; j < D; ++j) {
        q[j] = art.dof_state[((size_t)env * D + j) * 2];
        qd[j] = art.dof_state[((size_t)env * D + j) * 2 + 1];
        qs[j] = art.dof_position_setpoint[(size_t)env * D + j];
        qds[j] = art.dof_velocity_setpoint[(size_t)env * D + j];
    }
    if constexpr (EFFORT) {
        for (int j = 0; j < D; ++j) {
            if (!eff->effort_dof[j + 1]) continue;
            const float e = eff->effort[(size_t)env * D + j], E = eff->effort_limit[j + 1];
            qs[j] = E > 0.0f ? fminf(fmaxf(e, -E), E) : e;
        }
    }
    const V3 grav = ld3c(cfg.gravity);
    Derived d;
    for (int step = 0; step < cfg.physics_steps; ++step) {
        d = update_states(s);
        float ref[M];
        if (cfg.controller == AGX_CTRL_NONE) {
#pragma unroll
            for (int i = 0; i < M; ++i) ref[i] = act[i];
        } else {
            float wr[6];
            controller_wrench(cfg, s, d, p.g, act, wr);
#pragma unroll
            for (int i = 0; i < M; ++i) {
                float acc = 0.0f;
#pragma unroll
                for (int j = 0; j < 6; ++j) acc += cfg.alloc_pinv[i * 6 + j] * wr[j];
                ref[i] = acc;
            }
        }
#pragma unroll
        for (int i = 0; i < M; ++i) p.thrust[i] = motor_update(cfg, p.thrust[i], ref[i], p.tau_inc[i], p.tau_dec[i], p.k[i]);
        float vbn = norm3(d.vb);
        V3 df = neg(ld3c(cfg.drag_lin1) * d.vb) + neg(ld3c(cfg.drag_lin2) * vbn * d.vb);
        V3 wabs{fabsf(d.wb.x), fabsf(d.wb.y), fabsf(d.wb.z)};
        V3 dtq = neg(ld3c(cfg.drag_ang1) * d.wb) + neg(ld3c(cfg.drag_ang2) * wabs * d.wb);
        if (buf.disturbance) {
            const float* dp = buf.disturbance + (size_t)env * 6;
            df = df + ld3(dp);
            dtq = dtq + ld3(dp + 3);
        } else if (buf.dist_counter) {
            float d6[6];
            disturbance_env((uint32_t)(cfg.env_id_offset + env), *buf.dist_counter + buf.dist_offset + (uint32_t)step, cfg.dist_prob,
                            cfg.dist_max, (uint32_t)(cfg.dist_seed & 0xffffffffu), (uint32_t)(cfg.dist_seed >> 32), d6);
            df = df + V3{d6[0], d6[1], d6[2]};
            dtq = dtq + V3{d6[3], d6[4], d6[5]};
        }
        float a0[6];
        const bool last = step + 1 == cfg.physics_steps;
        float* imu = (IMU && last && (!JFORCE || imu_input)) ? imu_input + (size_t)env * 9 : nullptr;
        art_dynamics<NB, IMU, EFFORT, JFORCE, PRISM>(art, s, q, qd, qs, qds, cfg.dt, grav, M, p.thrust, quat_rotate(s.q, df),
                                                     quat_rotate(s.q, dtq), a0, qdd, imu_body, imu, eff,
                                                     (JFORCE && last) ? joint_wrench : nullptr, dof_force, pmask);
        art_integrate(cfg, art, s, a0, q, qd, qdd);
    }
    if (cfg.physics_steps == 0) d = update_states(s);
    if constexpr (JFORCE) {
        if (cfg.physics_steps == 0 && (!PRISM || joint_wrench)) {
            for (int k = 0; k < 6 * art.num_bodies; ++k) joint_wrench[k] = 0.0f;
            for (int j = 0; j < D; ++j) dof_force[j] = 0.0f;
        }
    }
    if constexpr (IMU) {
        if (cfg.physics_steps == 0 && (!JFORCE || imu_input)) {
            const V3 wb = art_body_angvel<NB, PRISM>(art, s, q, qd, imu_body, pmask);
            float* o = imu_input + (size_t)env * 9;
            o[0] = 0.0f; o[1] = 0.0f; o[2] = 0.0f; o[3] = 0.0f; o[4] = 0.0f; o[5] = 0.0f;
            o[6] = wb.x; o[7] = wb.y; o[8] = wb.z;
        }
    }
    float r[13];
    pack(s, r);
#pragma unroll
    for (int j = 0; j < 13; ++j) buf.root_state[(size_t)env * 13 + j] = r[j];
#pragma unroll
    for (int i = 0; i < M; ++i) buf.motor_thrust[(size_t)env * M + i] = p.thrust[i];
    for (int j = 0; j < D; ++j) {
        art.dof_state[((size_t)env * D + j) * 2] = q[j];
        art.dof_state[((size_t)env * D + j) * 2 + 1] = qd[j];
    }
    auto st3 = [&](float* a, V3 v) {
        if (a) { a[(size_t)env * 3] = v.x; a[(size_t)env * 3 + 1] = v.y; a[(size_t)env * 3 + 2] = v.z; }
    };
    st3(buf.euler, d.euler);
    if (buf.vehicle_orientation) {
        float* o = buf.vehicle_orientation + (size_t)env * 4;
        o[0] = d.qveh.x; o[1] = d.qveh.y; o[2] = d.qveh.z; o[3] = d.qveh.w;
    }
    st3(buf.vehicle_linvel, d.vveh);
    st3(buf.body_linvel, d.vb);
    st3(buf.body_angvel, d.wb);
}

// ---- per-body state of one env (agx_hp1_articulated_body_state) ------------------------------------------------------------
// rows [B][13]: body i's row at rows + 13 i, laid out like a root_state row (world position of the body-frame origin, xyzw quaternion
// body -> world, world linear velocity of the body-frame origin, world angular velocity).  root [13] = the env's root_state row, dof
// [D][2] = its (q, q-dot).  Row 0 is the root row, copied.  The forward kinematics are art_dynamics': R_i = R_l joint_R_i
// axis_angle(axis_i, q), P_i = P_l + R_l joint_p_i, V_i = V_l + S_i q-dot with S_i = (a, P_i x a), a = R_l joint_R_i axis_i.  The
// rows double as the scratch of the sweep (parent before child): while it runs, row i >= 1 holds (P_i relative to the base origin,
// quaternion of R_i, linear part of V_i = the velocity of the body point at the base origin, w_i), and R_l is rebuilt from row l's
// quaternion.  A last pass turns each row into world position x_0 + P_i and origin velocity V_lin + w_i x P_i.
// PRISM: the joint of every body i set in pmask is prismatic: R_i = R_l joint_R_i, P_i = P_l + R_l joint_p_i + a q, S_i = (0, a).
template <int NB, bool PRISM = false>
AGX_DEV void art_body_states(const AgxArticulation& art, const float* root, const float* dof, float* rows, uint32_t pmask = 0) {
    const int B = art.num_bodies;
#pragma unroll
    for (int k = 0; k < 13; ++k) rows[k] = root[k];
    for (int i = 1; i < NB; ++i) {
        if (i >= B) break;
        if constexpr (PRISM) {
            if ((pmask >> i) & 1u) {
                const int l = art.parent[i];
                const float* pl = rows + 13 * l;
                const M33 Rl = quat_to_matrix(Q4{pl[3], pl[4], pl[5], pl[6]});
                const V3 Pl = (l == 0) ? V3{0.0f, 0.0f, 0.0f} : ld3(pl);
                const M33 Ri = mul33(Rl, ld33(art.joint_R[i]));
                const V3 aw = mul33v(Ri, ld3(art.axis[i]));
                const float qi = dof[2 * (i - 1)], qd = dof[2 * (i - 1) + 1];
                const V3 Pi = Pl + mul33v(Rl, ld3(art.joint_p[i])) + aw * qi;
                const Q4 o = matrix_cols_to_quat(V3{Ri.m[0], Ri.m[3], Ri.m[6]}, V3{Ri.m[1], Ri.m[4], Ri.m[7]}, V3{Ri.m[2], Ri.m[5], Ri.m[8]});
                float* r = rows + 13 * i;
                r[0] = Pi.x; r[1] = Pi.y; r[2] = Pi.z;
                r[3] = o.x; r[4] = o.y; r[5] = o.z; r[6] = o.w;
                r[7] = pl[7] + aw.x * qd; r[8] = pl[8] + aw.y * qd; r[9] = pl[9] + aw.z * qd;
                r[10] = pl[10]; r[11] = pl[11]; r[12] = pl[12];
                continue;
            }
        }
        // the joint rotation first, while little else is live: sincosf's rarely taken wide-argument reduction then keeps its
        // six-word table in registers instead of a stack frame
        const V3 ax = ld3(art.axis[i]);
        const M33 Rq = axis_angle(ax, dof[2 * (i - 1)]);
        const int l = art.parent[i];
        const float* pl = rows + 13 * l;
        const M33 Rl = quat_to_matrix(Q4{pl[3], pl[4], pl[5], pl[6]});
        const V3 Pl = (l == 0) ? V3{0.0f, 0.0f, 0.0f} : ld3(pl);
        const M33 RJ = mul33(Rl, ld33(art.joint_R[i]));
        const M33 Ri = mul33(RJ, Rq);
        const V3 Pi = Pl + mul33v(Rl, ld3(art.joint_p[i]));
        const V3 aw = mul33v(RJ, ax);
        const V3 lin = cross(Pi, aw);
        const float qd = dof[2 * (i - 1) + 1];
        const Q4 qi = matrix_cols_to_quat(V3{Ri.m[0], Ri.m[3], Ri.m[6]}, V3{Ri.m[1], Ri.m[4], Ri.m[7]}, V3{Ri.m[2], Ri.m[5], Ri.m[8]});
        float* r = rows + 13 * i;
        r[0] = Pi.x; r[1] = Pi.y; r[2] = Pi.z;
        r[3] = qi.x; r[4] = qi.y; r[5] = qi.z; r[6] = qi.w;
        r[7] = pl[7] + lin.x * qd; r[8] = pl[8] + lin.y * qd; r[9] = pl[9] + lin.z * qd;
        r[10] = pl[10] + aw.x * qd; r[11] = pl[11] + aw.y * qd; r[12] = pl[12] + aw.z * qd;
    }
    const V3 x0 = ld3(rows);
    for (int i = 1; i < NB; ++i) {
        if (i >= B) break;
        float* r = rows + 13 * i;
        const V3 P = ld3(r);
        const V3 v = ld3(r + 7) + cross(ld3(r + 10), P);
        r[0] = x0.x + P.x; r[1] = x0.y + P.y; r[2] = x0.z + P.z;
        r[7] = v.x; r[8] = v.y; r[9] = v.z;
    }
}

}  // namespace agx
