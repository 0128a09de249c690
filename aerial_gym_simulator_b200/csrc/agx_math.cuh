// Device math helpers shared by the HP1 / HP2 kernels (xyzw quaternions).
// Each helper names the reference function whose arithmetic it follows
// (aerial_gym/utils/math.py); association order is kept where it is free to do so.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

// AGX_DEV: device-only in the product build.  tests/csrc/host_shadow.cu defines AGX_HOST_SHADOW to get the very same
// functions as host code, so per-env arithmetic can be checked against the oracle on a machine without a GPU.
#ifdef AGX_HOST_SHADOW
#include <math.h>
#define AGX_DEV __host__ __device__ __forceinline__
#else
#define AGX_DEV __device__ __forceinline__
#endif

namespace agx {

// sin/cos of an angle in [-2pi, 2pi].  AGX_FAST_TRIG: MUFU.SIN/COS (__sincosf, abs error <= 2^-21.4
// on [-pi, pi], CUDA C Programming Guide table 9) instead of the ~40-instruction libdevice path.
// Always inline: one shared out-of-line copy sends every value live across its calls through the stack, and in the HP1 step kernel
// that put local-memory traffic inside the physics sub-step loop (DESIGN 6).
#ifdef AGX_FAST_TRIG
AGX_DEV void sincos_(float x, float* s, float* c) { __sincosf(x, s, c); }
#else
AGX_DEV void sincos_(float x, float* s, float* c) { sincosf(x, s, c); }
#endif

// same idea for atan2f (two per update_states): -DAGX_HP1_NOINLINE_ATAN2, an experiment
#if defined(AGX_HP1_NOINLINE_ATAN2) && !defined(AGX_HOST_SHADOW)
__device__ __noinline__ float atan2_shared_(float y, float x) { return atan2f(y, x); }
AGX_DEV float atan2_(float y, float x) { return atan2_shared_(y, x); }
#else
AGX_DEV float atan2_(float y, float x) { return atan2f(y, x); }
#endif

#define AGX_PI_F 3.14159265358979323846f
#define AGX_TWO_PI_F 6.28318530717958647692f

struct V3 {
    float x, y, z;
};
struct Q4 {
    float x, y, z, w;
};

AGX_DEV V3 mk3(float x, float y, float z) { return V3{x, y, z}; }
AGX_DEV V3 operator+(V3 a, V3 b) { return V3{a.x + b.x, a.y + b.y, a.z + b.z}; }
AGX_DEV V3 operator-(V3 a, V3 b) { return V3{a.x - b.x, a.y - b.y, a.z - b.z}; }
AGX_DEV V3 operator*(V3 a, float s) { return V3{a.x * s, a.y * s, a.z * s}; }
AGX_DEV V3 operator*(V3 a, V3 b) { return V3{a.x * b.x, a.y * b.y, a.z * b.z}; }
AGX_DEV V3 neg(V3 a) { return V3{-a.x, -a.y, -a.z}; }
AGX_DEV float dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
AGX_DEV V3 cross(V3 a, V3 b) {
    return V3{a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
}
AGX_DEV float norm3(V3 a) { return sqrtf(dot(a, a)); }
AGX_DEV V3 ld3(const float* p) { return V3{p[0], p[1], p[2]}; }

// utils/math.py:58-65  quat_rotate
AGX_DEV V3 quat_rotate(Q4 q, V3 v) {
    V3 qv{q.x, q.y, q.z};
    float s = 2.0f * q.w * q.w - 1.0f;
    V3 a = v * s;
    V3 b = cross(qv, v) * q.w * 2.0f;
    V3 c = qv * dot(qv, v) * 2.0f;
    return a + b + c;
}
// utils/math.py:339-347  quat_rotate_inverse
AGX_DEV V3 quat_rotate_inverse(Q4 q, V3 v) {
    V3 qv{q.x, q.y, q.z};
    float s = 2.0f * q.w * q.w - 1.0f;
    V3 a = v * s;
    V3 b = cross(qv, v) * q.w * 2.0f;
    V3 c = qv * dot(qv, v) * 2.0f;
    return a - b + c;
}
// utils/math.py:313-320  quat_apply
AGX_DEV V3 quat_apply(Q4 q, V3 v) {
    V3 qv{q.x, q.y, q.z};
    V3 t = cross(qv, v) * 2.0f;
    return v + t * q.w + cross(qv, t);
}
AGX_DEV Q4 quat_conj(Q4 q) { return Q4{-q.x, -q.y, -q.z, q.w}; }

// utils/math.py:242-263  quat_mul (9-multiply form)
AGX_DEV Q4 quat_mul(Q4 a, Q4 b) {
    float ww = (a.z + a.x) * (b.x + b.y);
    float yy = (a.w - a.y) * (b.w + b.z);
    float zz = (a.w + a.y) * (b.w - b.z);
    float xx = ww + yy + zz;
    float qq = 0.5f * (xx + (a.z - a.x) * (b.x - b.y));
    Q4 r;
    r.w = qq - ww + (a.z - a.y) * (b.y - b.z);
    r.x = qq - xx + (a.x + a.w) * (b.x + b.w);
    r.y = qq - yy + (a.w - a.x) * (b.y + b.z);
    r.z = qq - zz + (a.z + a.y) * (b.w - b.x);
    return r;
}

struct M33 {
    float m[9];  // row-major
};
// utils/math.py:266-293  quat_to_rotation_matrix
AGX_DEV M33 quat_to_matrix(Q4 q) {
    float xx = q.x * q.x, xy = q.x * q.y, xz = q.x * q.z, xw = q.x * q.w;
    float yy = q.y * q.y, yz = q.y * q.z, yw = q.y * q.w;
    float zz = q.z * q.z, zw = q.z * q.w;
    M33 r;
    r.m[0] = 1.0f - 2.0f * (yy + zz);
    r.m[1] = 2.0f * (xy - zw);
    r.m[2] = 2.0f * (xz + yw);
    r.m[3] = 2.0f * (xy + zw);
    r.m[4] = 1.0f - 2.0f * (xx + zz);
    r.m[5] = 2.0f * (yz - xw);
    r.m[6] = 2.0f * (xz - yw);
    r.m[7] = 2.0f * (yz + xw);
    r.m[8] = 1.0f - 2.0f * (xx + yy);
    return r;
}

// python-style x % 2pi for x in (-2pi, 2pi): fmod is the identity there, then the sign fix.
AGX_DEV float wrap_0_2pi(float x) { return (x < 0.0f) ? x + AGX_TWO_PI_F : x; }
// utils/math.py:149-152 ssa for a in [0, 2pi): remainder(a + pi, 2pi) - pi
AGX_DEV float ssa_0_2pi(float a) {
    float t = a + AGX_PI_F;
    t = (t >= AGX_TWO_PI_F) ? t - AGX_TWO_PI_F : t;
    return t - AGX_PI_F;
}

// utils/math.py:123-146 get_euler_xyz_tensor: roll/pitch/yaw each wrapped to [0, 2pi)
AGX_DEV V3 euler_xyz_0_2pi(Q4 q) {
    float sinr_cosp = 2.0f * (q.w * q.x + q.y * q.z);
    float cosr_cosp = q.w * q.w - q.x * q.x - q.y * q.y + q.z * q.z;
    float roll = atan2_(sinr_cosp, cosr_cosp);
    float sinp = 2.0f * (q.w * q.y - q.z * q.x);
    float pitch = (fabsf(sinp) >= 1.0f) ? copysignf(0.5f * AGX_PI_F, sinp) : asinf(sinp);
    float siny_cosp = 2.0f * (q.w * q.z + q.x * q.y);
    float cosy_cosp = q.w * q.w + q.x * q.x - q.y * q.y - q.z * q.z;
    float yaw = atan2_(siny_cosp, cosy_cosp);
    return V3{wrap_0_2pi(roll), wrap_0_2pi(pitch), wrap_0_2pi(yaw)};
}

// utils/math.py:155-172 quat_from_euler_xyz
AGX_DEV Q4 quat_from_euler(float roll, float pitch, float yaw) {
    float sy, cy, sr, cr, sp, cp;
    sincos_(yaw * 0.5f, &sy, &cy);
    sincos_(roll * 0.5f, &sr, &cr);
    sincos_(pitch * 0.5f, &sp, &cp);
    Q4 q;
    q.w = cy * cr * cp + sy * sr * sp;
    q.x = cy * sr * cp - sy * cr * sp;
    q.y = cy * cr * sp + sy * sr * cp;
    q.z = sy * cr * cp - cy * sr * sp;
    return q;
}
// same with roll = pitch = 0 (vehicle_frame_quat_from_quat, utils/math.py:175-180):
// cos(0)=1, sin(0)=0 make the products exact, so only the yaw half-angle survives.
AGX_DEV Q4 quat_from_yaw(float yaw) {
    float sy, cy;
    sincos_(yaw * 0.5f, &sy, &cy);
    return Q4{0.0f, 0.0f, sy, cy};
}

// pytorch3d.transforms.matrix_to_quaternion (published algorithm) -> xyzw.
// R given by columns b1,b2,b3 (base_lee_controller.py:184-189).
AGX_DEV Q4 matrix_cols_to_quat(V3 b1, V3 b2, V3 b3) {
    float m00 = b1.x, m10 = b1.y, m20 = b1.z;
    float m01 = b2.x, m11 = b2.y, m21 = b2.z;
    float m02 = b3.x, m12 = b3.y, m22 = b3.z;
    float t0 = 1.0f + m00 + m11 + m22;
    float t1 = 1.0f + m00 - m11 - m22;
    float t2 = 1.0f - m00 + m11 - m22;
    float t3 = 1.0f - m00 - m11 + m22;
    float a0 = sqrtf(fmaxf(t0, 0.0f)), a1 = sqrtf(fmaxf(t1, 0.0f));
    float a2 = sqrtf(fmaxf(t2, 0.0f)), a3 = sqrtf(fmaxf(t3, 0.0f));
    // argmax, first index wins ties (torch.argmax)
    int idx = 0;
    float best = a0;
    if (a1 > best) { best = a1; idx = 1; }
    if (a2 > best) { best = a2; idx = 2; }
    if (a3 > best) { best = a3; idx = 3; }
    float den = 2.0f * fmaxf(best, 0.1f);
    float w, x, y, z;
    if (idx == 0) { w = a0 * a0; x = m21 - m12; y = m02 - m20; z = m10 - m01; }
    else if (idx == 1) { w = m21 - m12; x = a1 * a1; y = m10 + m01; z = m02 + m20; }
    else if (idx == 2) { w = m02 - m20; x = m10 + m01; y = a2 * a2; z = m12 + m21; }
    else { w = m10 - m01; x = m20 + m02; y = m21 + m12; z = a3 * a3; }
    return Q4{x / den, y / den, z / den, w / den};
}

// ---------------------------------------------------------------------------------------
// Philox4x32-10 counter-based RNG (Salmon et al. 2011) -- device-side reset sampling.
// Spec shared with oracle/philox.py: counter = (env_gid, episode, block, 0), key = seed.
// ---------------------------------------------------------------------------------------
struct U4 {
    uint32_t x, y, z, w;
};
AGX_DEV uint32_t mulhi32(uint32_t a, uint32_t b) {
#ifdef __CUDA_ARCH__
    return __umulhi(a, b);
#else
    return (uint32_t)(((uint64_t)a * (uint64_t)b) >> 32);
#endif
}
AGX_DEV U4 philox4x32_10(U4 ctr, uint32_t k0, uint32_t k1) {
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
    for (int i = 0; i < 10; ++i) {
        uint32_t hi0 = mulhi32(M0, ctr.x), lo0 = M0 * ctr.x;
        uint32_t hi1 = mulhi32(M1, ctr.z), lo1 = M1 * ctr.z;
        U4 n;
        n.x = hi1 ^ ctr.y ^ k0;
        n.y = lo1;
        n.z = hi0 ^ ctr.w ^ k1;
        n.w = lo0;
        ctr = n;
        k0 += W0;
        k1 += W1;
    }
    return ctr;
}
AGX_DEV float u01(uint32_t x) { return (float)(x >> 8) * (1.0f / 16777216.0f); }

}  // namespace agx
