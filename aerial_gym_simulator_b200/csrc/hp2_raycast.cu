// HP2: depth / segmentation / LiDAR ray-caster for sm_90a (H100).
//
//   agx_hp2_update_scene : per env (one CTA): instance transform of template triangles into
//                          world space, object AABBs, 30-bit Morton codes, bitonic sort in shared
//                          memory, implicit balanced binary BVH (heap order) bottom-up.
//   agx_hp2_cast         : persistent CTAs; a work item is one (env, sensor, row block).  The
//                          env's whole scene (BVH nodes + leaf map + triangle slabs) is staged
//                          into shared memory with TMA bulk copies (cp.async.bulk + mbarrier,
//                          SASS UBLKCP) when it fits (<= ~200 KB), else traversed from L2.
//                          Per ray: sensor pose compose, ray generation, stack traversal,
//                          Moller-Trumbore on the leaf's triangle slab, fused range-limit /
//                          normalise epilogue, coalesced row stores.
//   mesh objects          : (URDF <mesh> / <sphere>) one top-level leaf each, over a per-template BLAS whose boxes the scene
//                          update refits in world space; the cast walks it per ray (hp2_cast_kernel<SMEM, false, true>).
//
// This unit is compiled with -fmad=false and every fusable multiply-add on the RESULT path is an
// explicit fmaf(): the arithmetic is then bit-reproducible by oracle/hp2_oracle.c
// (-ffp-contract=off), so depth and segmentation are bit-identical to the brute-force oracle
// regardless of traversal order (ties on t resolve to the lowest triangle index in both).
// The AABB slab tests only cull, are padded, and need no bit contract.
//
// No tensor-core path: closest-hit traversal is divergent scalar FP32 work.
#include <cuda_runtime.h>
#include <float.h>
#include <stdint.h>

#include <type_traits>

#include "../../include/aerial_gym_b200.h"
#include "agx_common.cuh"
#include "contact_core.cuh"

namespace {

struct v3 {
    float x, y, z;
};
struct q4 {
    float x, y, z, w;
};

// ---- result-path arithmetic (bit contract with oracle/hp2_oracle.c) ----------------------
__device__ __forceinline__ float dot3(v3 a, v3 b) { return fmaf(a.z, b.z, fmaf(a.y, b.y, a.x * b.x)); }
__device__ __forceinline__ v3 cross3(v3 a, v3 b) {
    return v3{fmaf(a.y, b.z, -(a.z * b.y)), fmaf(a.z, b.x, -(a.x * b.z)), fmaf(a.x, b.y, -(a.y * b.x))};
}
__device__ __forceinline__ v3 sub3(v3 a, v3 b) { return v3{a.x - b.x, a.y - b.y, a.z - b.z}; }
__device__ __forceinline__ v3 normalize3(v3 a) {
    float n = sqrtf(dot3(a, a));
    return v3{a.x / n, a.y / n, a.z / n};
}
// warp quat_rotate == utils/math.py:58-65
__device__ __forceinline__ v3 quat_rotate(q4 q, v3 v) {
    v3 qv{q.x, q.y, q.z};
    float s = fmaf(2.0f * q.w, q.w, -1.0f);
    v3 c = cross3(qv, v);
    float d2 = 2.0f * dot3(qv, v);
    float w2 = 2.0f * q.w;
    return v3{fmaf(qv.x, d2, fmaf(c.x, w2, v.x * s)), fmaf(qv.y, d2, fmaf(c.y, w2, v.y * s)),
              fmaf(qv.z, d2, fmaf(c.z, w2, v.z * s))};
}
// utils/math.py:313-320 quat_apply
__device__ __forceinline__ v3 quat_apply(q4 q, v3 v) {
    v3 qv{q.x, q.y, q.z};
    v3 c = cross3(qv, v);
    v3 t{2.0f * c.x, 2.0f * c.y, 2.0f * c.z};
    v3 c2 = cross3(qv, t);
    return v3{fmaf(q.w, t.x, v.x) + c2.x, fmaf(q.w, t.y, v.y) + c2.y, fmaf(q.w, t.z, v.z) + c2.z};
}
// utils/math.py:242-263 quat_mul
__device__ __forceinline__ q4 quat_mul(q4 a, q4 b) {
    float ww = (a.z + a.x) * (b.x + b.y);
    float yy = (a.w - a.y) * (b.w + b.z);
    float zz = (a.w + a.y) * (b.w - b.z);
    float xx = ww + yy + zz;
    float qq = 0.5f * fmaf(a.z - a.x, b.x - b.y, xx);
    q4 r;
    r.w = fmaf(a.z - a.y, b.y - b.z, qq - ww);
    r.x = fmaf(a.x + a.w, b.x + b.w, qq - xx);
    r.y = fmaf(a.w - a.x, b.y + b.z, qq - yy);
    r.z = fmaf(a.z + a.y, b.w - b.x, qq - zz);
    return r;
}
__device__ __forceinline__ v3 kinv_mul(const float* k, v3 c) {
    return v3{fmaf(k[2], c.z, fmaf(k[1], c.y, k[0] * c.x)), fmaf(k[5], c.z, fmaf(k[4], c.y, k[3] * c.x)),
              fmaf(k[8], c.z, fmaf(k[7], c.y, k[6] * c.x))};
}

constexpr float kAabbPad = 1e-4f;  // metres; culling only
constexpr int kNodeFloats = 8;     // lo.xyz,0 | hi.xyz,0
constexpr int kTriFloats = 12;     // v0.xyz,seg | e1.xyz,0 | e2.xyz,0
constexpr int kObbFloats = 16;     // c.xyz | a0.xyz | a1.xyz | a2.xyz | half.xyz | valid

// =========================================================================================
// scene update: transform + BVH build, one CTA per env
// =========================================================================================
__device__ __forceinline__ uint32_t expand_bits10(uint32_t v) {
    v = (v * 0x00010001u) & 0xFF0000FFu;
    v = (v * 0x00000101u) & 0x0F00F00Fu;
    v = (v * 0x00000011u) & 0xC30C30C3u;
    v = (v * 0x00000005u) & 0x49249249u;
    return v;
}

__global__ void __launch_bounds__(256)
hp2_update_scene_kernel(const __grid_constant__ AgxHp2Scene sc, const uint8_t* __restrict__ mask) {
    const int e = blockIdx.x;
    if (mask && !mask[e]) return;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int K = sc.num_objects, P = sc.leaves_pow2, L = sc.tris_per_object;
    float* s_nodes = reinterpret_cast<float*>(smem_raw);                      // [(2P-1)*8]
    uint32_t* s_key = reinterpret_cast<uint32_t*>(s_nodes + (size_t)(2 * P) * kNodeFloats);  // [P]
    int32_t* s_val = reinterpret_cast<int32_t*>(s_key + P);                   // [P]
    float* s_olo = reinterpret_cast<float*>(s_val + P);                       // [K*3] object AABBs
    float* s_ohi = s_olo + (size_t)K * 3;
    const int tid = threadIdx.x, nt = blockDim.x;

    float* tris = sc.tris + (size_t)e * K * L * kTriFloats;
    // pass A: world-space triangle slabs (warp_env_manager.py:44-48 tf_apply over all vertices)
    for (int i = tid; i < K * L; i += nt) {
        int k = i / L, slot = i - k * L;
        const float* p = sc.obj_pose + ((size_t)e * K + k) * sc.obj_pose_stride;
        v3 t{p[0], p[1], p[2]};
        q4 q{p[3], p[4], p[5], p[6]};
        int tm = sc.obj_template[(size_t)e * K + k];
        int f0 = sc.tmpl_tri_offset[tm], f1 = sc.tmpl_tri_offset[tm + 1];
        float4 o0 = make_float4(0.f, 0.f, 0.f, __int_as_float(AGX_NO_HIT_SEG_VAL)), o1 = make_float4(0.f, 0.f, 0.f, 0.f), o2 = o1;
        if (f0 + slot < f1) {
            int f = f0 + slot;
            const float* tv = sc.tmpl_tris + (size_t)f * 9;
            v3 wa = quat_apply(q, v3{tv[0], tv[1], tv[2]});
            v3 wb = quat_apply(q, v3{tv[3], tv[4], tv[5]});
            v3 wc = quat_apply(q, v3{tv[6], tv[7], tv[8]});
            wa.x += t.x; wa.y += t.y; wa.z += t.z;
            wb.x += t.x; wb.y += t.y; wb.z += t.z;
            wc.x += t.x; wc.y += t.y; wc.z += t.z;
            v3 e1 = sub3(wb, wa), e2 = sub3(wc, wa);
            int seg = sc.tmpl_seg_base[f] + sc.obj_seg_counter[(size_t)e * K + k] * sc.tmpl_seg_mask[f];
            o0 = make_float4(wa.x, wa.y, wa.z, __int_as_float(seg));
            o1 = make_float4(e1.x, e1.y, e1.z, 0.f);
            o2 = make_float4(e2.x, e2.y, e2.z, 0.f);
        }
        float4* dst = reinterpret_cast<float4*>(tris + (size_t)i * kTriFloats);
        dst[0] = o0; dst[1] = o1; dst[2] = o2;
    }
    const int M = sc.num_meshes;
    const int32_t* slot = M ? sc.obj_mesh_slot + (size_t)e * K * 2 : nullptr;
    if (M) {  // mesh objects: world triangles into the env's mesh slab, in BLAS leaf order (same arithmetic as pass A)
        float* wt = sc.mesh_world_tris + (size_t)e * sc.mesh_tris_per_env * kTriFloats;
        for (int k = 0; k < K; ++k) {
            if (slot[2 * k] < 0) continue;
            const float* p = sc.obj_pose + ((size_t)e * K + k) * sc.obj_pose_stride;
            v3 t{p[0], p[1], p[2]};
            q4 q{p[3], p[4], p[5], p[6]};
            const int m = sc.tmpl_mesh[sc.obj_template[(size_t)e * K + k]];
            const int f0 = sc.mesh_tri_offset[m], n = sc.mesh_tri_offset[m + 1] - f0;
            const int seg = sc.mesh_seg[2 * m] + sc.obj_seg_counter[(size_t)e * K + k] * sc.mesh_seg[2 * m + 1];
            for (int i = tid; i < n; i += nt) {
                const float* tv = sc.mesh_tris + (size_t)(f0 + i) * 9;
                v3 wa = quat_apply(q, v3{tv[0], tv[1], tv[2]});
                v3 wb = quat_apply(q, v3{tv[3], tv[4], tv[5]});
                v3 wc = quat_apply(q, v3{tv[6], tv[7], tv[8]});
                wa.x += t.x; wa.y += t.y; wa.z += t.z;
                wb.x += t.x; wb.y += t.y; wb.z += t.z;
                wc.x += t.x; wc.y += t.y; wc.z += t.z;
                v3 e1 = sub3(wb, wa), e2 = sub3(wc, wa);
                float4* dst = reinterpret_cast<float4*>(wt + (size_t)(slot[2 * k] + i) * kTriFloats);
                dst[0] = make_float4(wa.x, wa.y, wa.z, __int_as_float(seg));
                dst[1] = make_float4(e1.x, e1.y, e1.z, __int_as_float(sc.mesh_tri_index[f0 + i]));
                dst[2] = make_float4(e2.x, e2.y, e2.z, 0.f);
            }
        }
    }
    if (sc.face_offset && tid == 0) {
        int acc = 0;
        for (int k = 0; k < K; ++k) {
            sc.face_offset[(size_t)e * K + k] = acc;
            int tm = sc.obj_template[(size_t)e * K + k];
            acc += min(L, sc.tmpl_tri_offset[tm + 1] - sc.tmpl_tri_offset[tm]);
            if (M && slot[2 * k] >= 0) acc += sc.mesh_tri_offset[sc.tmpl_mesh[tm] + 1] - sc.mesh_tri_offset[sc.tmpl_mesh[tm]];
        }
    }
    if (sc.obb) {  // world-frame oriented boxes of box-shaped objects (culling aid)
        for (int k = tid; k < K; k += nt) {
            const float* p = sc.obj_pose + ((size_t)e * K + k) * sc.obj_pose_stride;
            v3 t{p[0], p[1], p[2]};
            q4 q{p[3], p[4], p[5], p[6]};
            const float* to = sc.tmpl_obb + (size_t)sc.obj_template[(size_t)e * K + k] * kObbFloats;
            float* o = sc.obb + ((size_t)e * K + k) * kObbFloats;
            v3 c = quat_apply(q, v3{to[0], to[1], to[2]});
            v3 a0 = quat_apply(q, v3{to[3], to[4], to[5]});
            v3 a1 = quat_apply(q, v3{to[6], to[7], to[8]});
            v3 a2 = quat_apply(q, v3{to[9], to[10], to[11]});
            o[0] = c.x + t.x; o[1] = c.y + t.y; o[2] = c.z + t.z;
            o[3] = a0.x; o[4] = a0.y; o[5] = a0.z; o[6] = a1.x; o[7] = a1.y; o[8] = a1.z; o[9] = a2.x; o[10] = a2.y; o[11] = a2.z;
            o[12] = to[12]; o[13] = to[13]; o[14] = to[14];  // true half extents; users pad them (obb_pad)
            o[15] = to[15];
        }
    }
    __syncthreads();  // slabs of this CTA are read back below (same CTA wrote them)
    if (M) {  // refit the BLAS boxes of the mesh objects bottom-up, one depth level at a time (the reference's mesh.refit())
        const float* wt = sc.mesh_world_tris + (size_t)e * sc.mesh_tris_per_env * kTriFloats;
        float* wn = sc.mesh_world_nodes + (size_t)e * sc.mesh_nodes_per_env * kNodeFloats;
        for (int d = AGX_HP2_BLAS_MAX_DEPTH - 1; d >= 0; --d) {
            for (int k = 0; k < K; ++k) {
                if (slot[2 * k] < 0) continue;
                const int m = sc.tmpl_mesh[sc.obj_template[(size_t)e * K + k]];
                const int* lv = sc.mesh_levels + (size_t)m * (AGX_HP2_BLAS_MAX_DEPTH + 1);
                const int2* topo = reinterpret_cast<const int2*>(sc.mesh_topo) + sc.mesh_node_offset[m];
                const float* ot = wt + (size_t)slot[2 * k] * kTriFloats;
                float* on = wn + (size_t)slot[2 * k + 1] * kNodeFloats;
                for (int i = lv[d] + tid; i < lv[d + 1]; i += nt) {
                    const int2 tp = topo[i];
                    float lo[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, hi[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
                    if (tp.y > 0) {
                        for (int s = tp.x; s < tp.x + tp.y; ++s) {
                            const float4* src = reinterpret_cast<const float4*>(ot + (size_t)s * kTriFloats);
                            float4 a = src[0], b = src[1], c = src[2];
                            float vx[3] = {a.x, a.x + b.x, a.x + c.x}, vy[3] = {a.y, a.y + b.y, a.y + c.y}, vz[3] = {a.z, a.z + b.z, a.z + c.z};
#pragma unroll
                            for (int j = 0; j < 3; ++j) {
                                lo[0] = fminf(lo[0], vx[j]); hi[0] = fmaxf(hi[0], vx[j]);
                                lo[1] = fminf(lo[1], vy[j]); hi[1] = fmaxf(hi[1], vy[j]);
                                lo[2] = fminf(lo[2], vz[j]); hi[2] = fmaxf(hi[2], vz[j]);
                            }
                        }
#pragma unroll
                        for (int j = 0; j < 3; ++j) {
                            float pad = kAabbPad + 1e-6f * fmaxf(fabsf(lo[j]), fabsf(hi[j]));
                            lo[j] -= pad;
                            hi[j] += pad;
                        }
                    } else {
                        const float* a = on + (size_t)tp.x * kNodeFloats;
                        const float* b = a + kNodeFloats;
#pragma unroll
                        for (int j = 0; j < 3; ++j) { lo[j] = fminf(a[j], b[j]); hi[j] = fmaxf(a[4 + j], b[4 + j]); }
                    }
                    float4* dst = reinterpret_cast<float4*>(on + (size_t)i * kNodeFloats);
                    dst[0] = make_float4(lo[0], lo[1], lo[2], 0.f);
                    dst[1] = make_float4(hi[0], hi[1], hi[2], 0.f);
                }
            }
            __syncthreads();
        }
    }
    // pass B: object AABBs from the slabs just written (a mesh object: its BLAS root box, already padded)
    for (int k = tid; k < K; k += nt) {
        if (M && slot[2 * k] >= 0) {
            const float* rn = sc.mesh_world_nodes + ((size_t)e * sc.mesh_nodes_per_env + slot[2 * k + 1]) * kNodeFloats;
#pragma unroll
            for (int j = 0; j < 3; ++j) { s_olo[k * 3 + j] = rn[j]; s_ohi[k * 3 + j] = rn[4 + j]; }
            continue;
        }
        float lo[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, hi[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
        int tm = sc.obj_template[(size_t)e * K + k];
        int n = min(L, sc.tmpl_tri_offset[tm + 1] - sc.tmpl_tri_offset[tm]);
        for (int s = 0; s < n; ++s) {
            const float4* src = reinterpret_cast<const float4*>(tris + ((size_t)k * L + s) * kTriFloats);
            float4 a = src[0], b = src[1], c = src[2];
            float vx[3] = {a.x, a.x + b.x, a.x + c.x}, vy[3] = {a.y, a.y + b.y, a.y + c.y}, vz[3] = {a.z, a.z + b.z, a.z + c.z};
#pragma unroll
            for (int j = 0; j < 3; ++j) {
                lo[0] = fminf(lo[0], vx[j]); hi[0] = fmaxf(hi[0], vx[j]);
                lo[1] = fminf(lo[1], vy[j]); hi[1] = fmaxf(hi[1], vy[j]);
                lo[2] = fminf(lo[2], vz[j]); hi[2] = fmaxf(hi[2], vz[j]);
            }
        }
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            float pad = kAabbPad + 1e-6f * fmaxf(fabsf(lo[j]), fabsf(hi[j]));
            s_olo[k * 3 + j] = lo[j] - pad;
            s_ohi[k * 3 + j] = hi[j] + pad;
        }
    }
    __syncthreads();
    // Morton keys over the env bounds (parked objects at -1000 clamp to a corner)
    float bl[3], bh[3];
    if (sc.bounds_min && sc.bounds_max) {
#pragma unroll
        for (int j = 0; j < 3; ++j) { bl[j] = sc.bounds_min[(size_t)e * 3 + j]; bh[j] = sc.bounds_max[(size_t)e * 3 + j]; }
    } else {
#pragma unroll
        for (int j = 0; j < 3; ++j) { bl[j] = -16.0f; bh[j] = 16.0f; }
    }
    for (int i = tid; i < P; i += nt) {
        uint32_t key = 0xFFFFFFFFu;
        int val = -1;
        if (i < K) {
            uint32_t c[3];
#pragma unroll
            for (int j = 0; j < 3; ++j) {
                float ctr = 0.5f * (s_olo[i * 3 + j] + s_ohi[i * 3 + j]);
                float u = (ctr - bl[j]) / fmaxf(bh[j] - bl[j], 1e-6f);
                u = fminf(fmaxf(u, 0.0f), 1.0f);
                c[j] = (uint32_t)fminf(u * 1023.0f, 1023.0f);
            }
            key = (expand_bits10(c[0]) << 2) | (expand_bits10(c[1]) << 1) | expand_bits10(c[2]);
            val = i;
        }
        s_key[i] = key;
        s_val[i] = val;
    }
    __syncthreads();
    // bitonic sort of (key, val) -- P is a power of two; ties broken by val for determinism
    for (int k2 = 2; k2 <= P; k2 <<= 1) {
        for (int j = k2 >> 1; j > 0; j >>= 1) {
            for (int i = tid; i < P; i += nt) {
                int ixj = i ^ j;
                if (ixj > i) {
                    uint32_t ka = s_key[i], kb = s_key[ixj];
                    int va = s_val[i], vb = s_val[ixj];
                    bool a_gt_b = (ka > kb) || (ka == kb && (uint32_t)va > (uint32_t)vb);
                    bool up = ((i & k2) == 0);
                    if (a_gt_b == up) {
                        s_key[i] = kb; s_key[ixj] = ka;
                        s_val[i] = vb; s_val[ixj] = va;
                    }
                }
            }
            __syncthreads();
        }
    }
    // leaves (heap index P-1+i)
    for (int i = tid; i < P; i += nt) {
        int obj = s_val[i];
        float* nd = s_nodes + (size_t)(P - 1 + i) * kNodeFloats;
        if (obj >= 0) {
            nd[0] = s_olo[obj * 3]; nd[1] = s_olo[obj * 3 + 1]; nd[2] = s_olo[obj * 3 + 2]; nd[3] = 0.f;
            nd[4] = s_ohi[obj * 3]; nd[5] = s_ohi[obj * 3 + 1]; nd[6] = s_ohi[obj * 3 + 2]; nd[7] = 0.f;
        } else {
            nd[0] = nd[1] = nd[2] = FLT_MAX; nd[3] = 0.f;
            nd[4] = nd[5] = nd[6] = -FLT_MAX; nd[7] = 0.f;
        }
    }
    __syncthreads();
    // internal levels bottom-up
    for (int width = P >> 1; width >= 1; width >>= 1) {
        for (int i = tid; i < width; i += nt) {
            int n = width - 1 + i;
            const float* a = s_nodes + (size_t)(2 * n + 1) * kNodeFloats;
            const float* b = s_nodes + (size_t)(2 * n + 2) * kNodeFloats;
            float* d = s_nodes + (size_t)n * kNodeFloats;
            d[0] = fminf(a[0], b[0]); d[1] = fminf(a[1], b[1]); d[2] = fminf(a[2], b[2]); d[3] = 0.f;
            d[4] = fmaxf(a[4], b[4]); d[5] = fmaxf(a[5], b[5]); d[6] = fmaxf(a[6], b[6]); d[7] = 0.f;
        }
        __syncthreads();
    }
    float* gn = sc.nodes + (size_t)e * (2 * P - 1) * kNodeFloats;
    for (int i = tid; i < (2 * P - 1) * kNodeFloats; i += nt) gn[i] = s_nodes[i];
    const int leaf_stride = P < 4 ? 4 : P;
    int32_t* gl = sc.leaf_object + (size_t)e * leaf_stride;
    for (int i = tid; i < leaf_stride; i += nt) gl[i] = (i < P) ? s_val[i] : -1;
}

// =========================================================================================
// ray casting
// =========================================================================================
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
// bounded spin: a mis-programmed copy must trap, never hang the GPU
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    for (uint32_t spin = 0; spin < (1u << 24); ++spin)
        if (mbar_try_wait(bar, parity)) return;
    __trap();
}
// TMA 1-D bulk copy global -> shared, completion on mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void tma_bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

struct Hit {
    float t;
    int tri;   // tie-break index: obj * L + slot, or (scenes with mesh objects) the face id in the env's concatenated mesh
};
struct MeshHit : Hit {
    int slab;  // >= 0 cluster slab index, < 0 mesh slab -(slab + 1)
};

// per-env view of the mesh objects of a scene (num_meshes > 0)
struct MeshCtx {
    const int32_t* slot;          // [K,2] first triangle / node in the env's mesh slabs, -1 = cluster object
    const int32_t* obj_template;  // [K]
    const int32_t* face_offset;   // [K]
    const float* tris;            // env mesh slab
    const float* nodes;           // env BLAS boxes
};
__device__ __forceinline__ MeshCtx mesh_ctx(const AgxHp2Scene& sc, int e) {
    const int K = sc.num_objects;
    return MeshCtx{sc.obj_mesh_slot + (size_t)e * K * 2, sc.obj_template + (size_t)e * K, sc.face_offset + (size_t)e * K,
                   sc.mesh_world_tris + (size_t)e * sc.mesh_tris_per_env * kTriFloats,
                   sc.mesh_world_nodes + (size_t)e * sc.mesh_nodes_per_env * kNodeFloats};
}
// triangle slab of a hit
template <bool MESH, class H>
__device__ __forceinline__ const float* hit_slab(const H& h, const float* tris, const MeshCtx& mc) {
    if constexpr (MESH) return h.slab >= 0 ? tris + (size_t)h.slab * kTriFloats : mc.tris + (size_t)(-h.slab - 1) * kTriFloats;
    else return tris + (size_t)h.tri * kTriFloats;
}

// Moller-Trumbore on one triangle slab (bit contract with oracle closest_hit)
__device__ __forceinline__ void tri_test(const float4* __restrict__ tp, int tri_index, v3 o, v3 d, float max_t, Hit& best) {
    float4 a = tp[0], b = tp[1], c = tp[2];
    v3 v0{a.x, a.y, a.z}, e1{b.x, b.y, b.z}, e2{c.x, c.y, c.z};
    v3 pv = cross3(d, e2);
    float det = dot3(e1, pv);
    if (fabsf(det) < 1e-20f) return;
    float inv = 1.0f / det;
    v3 tv = sub3(o, v0);
    float u = dot3(tv, pv) * inv;
    if (u < 0.0f || u > 1.0f) return;
    v3 qv = cross3(tv, e1);
    float v = dot3(d, qv) * inv;
    if (v < 0.0f || u + v > 1.0f) return;
    float t = dot3(e2, qv) * inv;
    if (t < 0.0f || !(t < max_t)) return;
    if (t < best.t || (t == best.t && tri_index < best.tri)) {
        best.t = t;
        best.tri = tri_index;
    }
}

// conservative slab test; returns entry distance or a negative value for a miss
__device__ __forceinline__ float aabb_entry(const float* nd, v3 o, v3 inv, float t_limit) {
    float4 lo = *reinterpret_cast<const float4*>(nd);
    float4 hi = *reinterpret_cast<const float4*>(nd + 4);
    float tx1 = (lo.x - o.x) * inv.x, tx2 = (hi.x - o.x) * inv.x;
    float ty1 = (lo.y - o.y) * inv.y, ty2 = (hi.y - o.y) * inv.y;
    float tz1 = (lo.z - o.z) * inv.z, tz2 = (hi.z - o.z) * inv.z;
    float tmin = fmaxf(fmaxf(fminf(tx1, tx2), fminf(ty1, ty2)), fmaxf(fminf(tz1, tz2), 0.0f));
    float tmax = fminf(fminf(fmaxf(tx1, tx2), fmaxf(ty1, ty2)), fmaxf(tz1, tz2));
    float slack = 1e-5f * (1.0f + fabsf(tmax));
    bool hit = (tmin <= tmax + slack) && (tmin <= t_limit + 1e-5f * (1.0f + t_limit));
    return hit ? tmin : -1.0f;
}

// padding of an oriented box for culling decisions: conservative, never culls a true hit
__device__ __forceinline__ float obb_pad(const float* __restrict__ b) {
    return 2e-4f + 4e-6f * (fabsf(b[0]) + fabsf(b[1]) + fabsf(b[2]) + b[12] + b[13] + b[14]);
}

// ray vs padded oriented box (object frame slabs); culling only
__device__ __forceinline__ bool obb_may_hit(const float* __restrict__ b, v3 o, v3 d, float t_limit) {
    v3 r{o.x - b[0], o.y - b[1], o.z - b[2]};
    const float pad = obb_pad(b);
    float tmin = 0.0f, tmax = t_limit + 1e-5f * (1.0f + t_limit);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float ax = b[3 + 3 * a], ay = b[4 + 3 * a], az = b[5 + 3 * a];
        const float oa = r.x * ax + r.y * ay + r.z * az;
        const float da = d.x * ax + d.y * ay + d.z * az;
        const float h = b[12 + a] + pad;
        if (fabsf(da) < 1e-12f) {
            if (fabsf(oa) > h) return false;
        } else {
            const float inv = 1.0f / da;
            float t1 = (-h - oa) * inv, t2 = (h - oa) * inv;
            tmin = fmaxf(tmin, fminf(t1, t2));
            tmax = fminf(tmax, fmaxf(t1, t2));
        }
    }
    return tmin <= tmax + 1e-5f * (1.0f + fabsf(tmax));
}

// one mesh object: walk its BLAS in world space (L2 reads); keys are face ids, so ties go to the lowest file-order index
__device__ __forceinline__ void mesh_object_test(const AgxHp2Scene& sc, const MeshCtx& mc, int obj, v3 o, v3 d, v3 inv, float max_t,
                                                 MeshHit& best) {
    const int ts = mc.slot[2 * obj];
    const int m = sc.tmpl_mesh[mc.obj_template[obj]];
    const int2* topo = reinterpret_cast<const int2*>(sc.mesh_topo) + sc.mesh_node_offset[m];
    const float* nodes = mc.nodes + (size_t)mc.slot[2 * obj + 1] * kNodeFloats;
    const float4* tp = reinterpret_cast<const float4*>(mc.tris + (size_t)ts * kTriFloats);
    const int fo = mc.face_offset[obj];
    int stack[AGX_HP2_BLAS_MAX_DEPTH];
    int sp = 0, node = 0;  // the root box is the object's top-level leaf box, already tested
    while (true) {
        const int2 t = topo[node];
        if (t.y > 0) {
            for (int s = t.x; s < t.x + t.y; ++s) {
                const int before = best.tri;
                tri_test(tp + 3 * s, fo + __float_as_int(tp[3 * s + 1].w), o, d, max_t, best);
                if (best.tri != before) best.slab = -(ts + s) - 1;
            }
            if (sp == 0) break;
            node = stack[--sp];
            continue;
        }
        const int c0 = t.x, c1 = c0 + 1;
        const float t0 = aabb_entry(nodes + (size_t)c0 * kNodeFloats, o, inv, best.t);
        const float t1 = aabb_entry(nodes + (size_t)c1 * kNodeFloats, o, inv, best.t);
        if (t0 >= 0.0f && t1 >= 0.0f) {
            if (t0 <= t1) { stack[sp++] = c1; node = c0; }
            else { stack[sp++] = c0; node = c1; }
        } else if (t0 >= 0.0f) {
            node = c0;
        } else if (t1 >= 0.0f) {
            node = c1;
        } else {
            if (sp == 0) break;
            node = stack[--sp];
        }
    }
}

// MESH: the scene has mesh objects (sc, mc given): their leaves walk the object's BLAS, cluster leaves key their triangles
// by face id so that ties resolve as in the env's concatenated mesh
template <bool SMEM, bool MESH = false>
__device__ __forceinline__ auto traverse(const float* __restrict__ nodes, const int32_t* __restrict__ leaf_obj,
                                         const float* __restrict__ tris, const float* __restrict__ obb, int P, int L, v3 o, v3 d,
                                         float max_t, const AgxHp2Scene* sc = nullptr, const MeshCtx* mc = nullptr) {
    typename std::conditional<MESH, MeshHit, Hit>::type best{};
    best.t = max_t;
    best.tri = 0x7fffffff;
    v3 inv{1.0f / d.x, 1.0f / d.y, 1.0f / d.z};
    int stack[24];
    int sp = 0;
    int node = 0;
    if (P == 1) {
        node = 0;
    } else if (aabb_entry(nodes, o, inv, best.t) < 0.0f) {
        return best;
    }
    while (true) {
        if (node >= P - 1) {  // leaf
            int obj = leaf_obj[node - (P - 1)];
            if constexpr (MESH) {
                if (obj >= 0 && mc->slot[2 * obj] >= 0) {
                    mesh_object_test(*sc, *mc, obj, o, d, inv, max_t, best);
                } else if (obj >= 0) {
                    const float4* tp = reinterpret_cast<const float4*>(tris + (size_t)obj * L * kTriFloats);
                    const int fo = mc->face_offset[obj];
                    for (int s = 0; s < L; ++s) {
                        const int before = best.tri;
                        tri_test(tp + 3 * s, fo + s, o, d, max_t, best);
                        if (best.tri != before) best.slab = obj * L + s;
                    }
                }
                obj = -1;
            }
            if (obj >= 0) {
                bool test = true;
                if (obb) {
                    const float* b = obb + (size_t)obj * kObbFloats;
                    if (b[15] != 0.0f) test = obb_may_hit(b, o, d, best.t);
                }
                if (test) {
                    const float4* tp = reinterpret_cast<const float4*>(tris + (size_t)obj * L * kTriFloats);
                    for (int s = 0; s < L; ++s) tri_test(tp + 3 * s, obj * L + s, o, d, max_t, best);
                }
            }
            if (sp == 0) break;
            node = stack[--sp];
            continue;
        }
        int c0 = 2 * node + 1, c1 = c0 + 1;
        float t0 = aabb_entry(nodes + (size_t)c0 * kNodeFloats, o, inv, best.t);
        float t1 = aabb_entry(nodes + (size_t)c1 * kNodeFloats, o, inv, best.t);
        if (t0 >= 0.0f && t1 >= 0.0f) {
            if (t0 <= t1) { stack[sp++] = c1; node = c0; }
            else { stack[sp++] = c0; node = c1; }
        } else if (t0 >= 0.0f) {
            node = c0;
        } else if (t1 >= 0.0f) {
            node = c1;
        } else {
            if (sp == 0) break;
            node = stack[--sp];
        }
    }
    return best;
}

// =========================================================================================
// Tile path (scenes of <= 128 leaf slots staged in shared memory): one warp = one 8x4 pixel tile.
//  1. the warp culls the scene's objects against the tile's ray bundle ONCE (lane j tests leaf slots
//     j, j+32, ...): four planes through the common ray origin spanned by the tile's corner rays, each
//     pushed out to the minimum of n.d over the 32 actual ray directions, so the test is conservative
//     for any ray set (camera pixels, LiDAR table entries, clamped border lanes);
//  2. every lane then tests its own ray against the few surviving candidates in the same order --
//     uniform control flow, no stack.  A canonical box (box_triangles order, obb[15] == 2) whose face
//     the ray enters well inside needs only that face's two triangles; everything else runs all L.
// The closest hit is the minimum over exact Moller-Trumbore tests with the oracle's tie-break, so the
// result is independent of candidate order and bit-identical to the brute-force oracle.
// =========================================================================================
__device__ __forceinline__ float warp_min_f(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ float warp_max_f(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ v3 shfl3(v3 a, int src) {
    return v3{__shfl_sync(0xffffffffu, a.x, src), __shfl_sync(0xffffffffu, a.y, src), __shfl_sync(0xffffffffu, a.z, src)};
}

constexpr int kTileMaxLeaves = 128;
constexpr int kBigSceneRecords = 384;  // record slots of the <false, true> tile path (43 KB of shared memory per CTA)
// per-image object record (shared memory, built once per work item by build_records):
//   [0..8] box axes A0 A1 A2 | [9..11] (o - c).A_k for the sensor origin o | [12..14] true half extents |
//   [15] pad | [16] kind (0 generic mesh in its AABB, 1 box-shaped bound only, 2 canonical box) | [17] object index |
//   [18] face-shortcut margin | [19] nearest possible hit distance | [20] farthest point distance
// 28-float stride: 8 lanes x 16 B of a float4 load hit 8 distinct bank groups (28 j mod 32 = 0,28,24,...,4)
constexpr int kRecFloats = 28;

// frustum: optional 4 inward plane normals through o that bound every ray of the work item (camera pixel
// blocks: ray directions are affine in the pixel coordinates before normalisation, so the block's corner
// rays span all of them); objects entirely outside one plane get no record.
__device__ __forceinline__ void build_records(const float* __restrict__ nodes, const int32_t* __restrict__ leaf,
                                              const float* __restrict__ obb, int P, v3 o, const v3* frustum, float t_far,
                                              float* __restrict__ rec, int* n_rec, int cap) {
    for (int slot = threadIdx.x; slot < P; slot += blockDim.x) {
        const int obj = leaf[slot];
        if (obj < 0) continue;
        v3 c, h, a0{1.f, 0.f, 0.f}, a1{0.f, 1.f, 0.f}, a2{0.f, 0.f, 1.f};
        float kind = 0.0f, pad;
        const float* b = obb ? obb + (size_t)obj * kObbFloats : nullptr;
        if (b && b[15] != 0.0f) {
            c = v3{b[0], b[1], b[2]};
            a0 = v3{b[3], b[4], b[5]}; a1 = v3{b[6], b[7], b[8]}; a2 = v3{b[9], b[10], b[11]};
            h = v3{b[12], b[13], b[14]};
            kind = b[15];
            pad = obb_pad(b);
        } else {  // generic template: the leaf's world AABB
            const float* nd = nodes + (size_t)(P - 1 + slot) * kNodeFloats;
            c = v3{0.5f * (nd[0] + nd[4]), 0.5f * (nd[1] + nd[5]), 0.5f * (nd[2] + nd[6])};
            h = v3{0.5f * (nd[4] - nd[0]), 0.5f * (nd[5] - nd[1]), 0.5f * (nd[6] - nd[2])};
            pad = 2e-4f + 4e-6f * (fabsf(nd[0]) + fabsf(nd[1]) + fabsf(nd[2]) + fabsf(nd[4]) + fabsf(nd[5]) + fabsf(nd[6]));
        }
        const v3 r = sub3(o, c);
        const float dist_c = sqrtf(dot3(r, r));
        const v3 hp{h.x + pad, h.y + pad, h.z + pad};
        const float rad_s = sqrtf(dot3(hp, hp));
        if (dist_c - rad_s > t_far * (1.0f + 1e-5f) + 1e-5f) continue;  // out of range for every ray of the item
        if (frustum) {
            bool outside = false;
            const v3 rc{-r.x, -r.y, -r.z};
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const v3 n = frustum[i];
                const float sN = dot3(n, rc);
                const float rad = fmaf(fabsf(dot3(n, a2)), hp.z, fmaf(fabsf(dot3(n, a1)), hp.y, fabsf(dot3(n, a0)) * hp.x));
                // rays satisfy n.d >= -1e-5 |n| (rounding of the corner rays): points on them n.x >= -1e-5 |n| |x|
                const float bound = -1e-5f * sqrtf(dot3(n, n)) * (dist_c + rad_s);
                if (sN + rad < bound - 1e-4f * (fabsf(sN) + rad + fabsf(bound))) outside = true;
            }
            if (outside) continue;
        }
        const int idx = atomicAdd(n_rec, 1);
        if (idx >= cap) continue;  // more survivors than record slots: the caller sees *n_rec > cap and walks the BVH per ray instead
        float* q = rec + (size_t)idx * kRecFloats;
        q[0] = a0.x; q[1] = a0.y; q[2] = a0.z; q[3] = a1.x; q[4] = a1.y; q[5] = a1.z; q[6] = a2.x; q[7] = a2.y; q[8] = a2.z;
        q[9] = dot3(r, a0); q[10] = dot3(r, a1); q[11] = dot3(r, a2);
        q[12] = h.x; q[13] = h.y; q[14] = h.z;
        q[15] = pad;
        q[16] = kind;
        q[17] = __int_as_float(obj);
        q[18] = 1e-3f * (1.0f + 0.05f * (fabsf(r.x) + fabsf(r.y) + fabsf(r.z)));
        q[19] = dist_c - rad_s;
        q[20] = dist_c + rad_s;
    }
}

struct TilePlanes {
    v3 n[4];
    float m[4];
    float t_far;
};
// four planes through the common ray origin spanned by the tile's corner rays (lanes 0, 7, 31, 24), each
// pushed out to the minimum of n.d over the 32 actual ray directions: conservative for any ray set
__device__ __forceinline__ TilePlanes tile_planes(v3 d, float max_t) {
    TilePlanes tp;
    const v3 c0 = shfl3(d, 0), c1 = shfl3(d, 7), c2 = shfl3(d, 31), c3 = shfl3(d, 24);
    const v3 dc{c0.x + c1.x + c2.x + c3.x, c0.y + c1.y + c2.y + c3.y, c0.z + c1.z + c2.z + c3.z};
    tp.n[0] = cross3(c0, c1); tp.n[1] = cross3(c1, c2); tp.n[2] = cross3(c2, c3); tp.n[3] = cross3(c3, c0);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        if (dot3(tp.n[i], dc) < 0.0f) tp.n[i] = v3{-tp.n[i].x, -tp.n[i].y, -tp.n[i].z};
        tp.m[i] = warp_min_f(dot3(tp.n[i], d));  // every ray of the tile satisfies n_i . d >= m_i
    }
    tp.t_far = warp_max_f(max_t);
    return tp;
}
// can any ray of the tile hit this object's (padded) box?
__device__ __forceinline__ bool tile_may_hit(const TilePlanes& tp, const float* __restrict__ q) {
    const float4 q0 = reinterpret_cast<const float4*>(q)[0], q1 = reinterpret_cast<const float4*>(q)[1];
    const float4 q2 = reinterpret_cast<const float4*>(q)[2], q3 = reinterpret_cast<const float4*>(q)[3];
    const float4 q4 = reinterpret_cast<const float4*>(q)[4], q5 = reinterpret_cast<const float4*>(q)[5];
    const v3 a0{q0.x, q0.y, q0.z}, a1{q0.w, q1.x, q1.y}, a2{q1.z, q1.w, q2.x};
    const float oa0 = q2.y, oa1 = q2.z, oa2 = q2.w;
    const float pad = q3.w;
    const float h0 = q3.x + pad, h1 = q3.y + pad, h2 = q3.z + pad;
    bool cand = q4.w <= tp.t_far * (1.0f + 1e-5f) + 1e-5f;  // nearest possible hit within range
    const float reach = q5.x;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float n0 = dot3(tp.n[i], a0), n1 = dot3(tp.n[i], a1), n2 = dot3(tp.n[i], a2);
        const float sN = -fmaf(oa2, n2, fmaf(oa1, n1, oa0 * n0));  // n . (c - o)
        const float rad = fmaf(fabsf(n2), h2, fmaf(fabsf(n1), h1, fabsf(n0) * h0));
        const float bound = tp.m[i] < 0.0f ? tp.m[i] * reach : 0.0f;
        if (sN + rad < bound - 1e-4f * (fabsf(sN) + rad + fabsf(bound))) cand = false;  // whole box outside plane i
    }
    return cand;
}

__constant__ unsigned char kBoxFaceTris[6][2] = {{0, 2}, {10, 11}, {1, 5}, {7, 9}, {3, 8}, {4, 6}};  // hp2.py box_triangles

// one ray (origin o, unit direction d) vs the object of record q
__device__ __forceinline__ void record_object_test(const float* __restrict__ q, const float* __restrict__ tris, int L, v3 o, v3 d,
                                                   float max_t, Hit& best) {
    const float4 q0 = reinterpret_cast<const float4*>(q)[0], q1 = reinterpret_cast<const float4*>(q)[1];
    const float4 q2 = reinterpret_cast<const float4*>(q)[2], q3 = reinterpret_cast<const float4*>(q)[3];
    const float4 q4 = reinterpret_cast<const float4*>(q)[4];
    const float oa[3] = {q2.y, q2.z, q2.w};
    const float hh[3] = {q3.x, q3.y, q3.z};
    const float pad = q3.w;
    const float da[3] = {fmaf(d.z, q0.z, fmaf(d.y, q0.y, d.x * q0.x)), fmaf(d.z, q1.y, fmaf(d.y, q1.x, d.x * q0.w)),
                         fmaf(d.z, q2.x, fmaf(d.y, q1.w, d.x * q1.z))};
    float te[3];
    float tmin = 0.0f, tmax = best.t + 1e-5f * (1.0f + best.t);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        te[a] = -FLT_MAX;
        if (fabsf(da[a]) < 1e-12f) {
            if (fabsf(oa[a]) > hh[a] + pad) return;
        } else {
            const float inv = __frcp_rn(da[a]);
            const float hp = hh[a] + pad;
            const float t1 = (-hp - oa[a]) * inv, t2 = (hp - oa[a]) * inv;
            tmin = fmaxf(tmin, fminf(t1, t2));
            tmax = fminf(tmax, fmaxf(t1, t2));
            te[a] = ((da[a] > 0.0f ? -hh[a] : hh[a]) - oa[a]) * inv;  // entry through the TRUE face plane of this axis
        }
    }
    if (!(tmin <= tmax + 1e-5f * (1.0f + fabsf(tmax)))) return;  // misses the padded box, or it lies beyond the best hit
    const int obj = __float_as_int(q4.y);
    const float4* tp = reinterpret_cast<const float4*>(tris + (size_t)obj * L * kTriFloats);
    const int tri0 = obj * L;
    if (q4.x == 2.0f && L >= 12) {
        // entry face = the axis entered last; valid shortcut only if the ray crosses that face well inside it
        const float t = fmaxf(te[0], fmaxf(te[1], te[2]));
        const bool a0 = te[0] >= te[1] && te[0] >= te[2], a1 = !a0 && te[1] >= te[2];  // selected axis (no dynamic indexing)
        const float da_sel = a0 ? da[0] : (a1 ? da[1] : da[2]);
        const float margin = q4.z;
        const bool lat0 = fabsf(fmaf(t, da[0], oa[0])) <= hh[0] - margin;
        const bool lat1 = fabsf(fmaf(t, da[1], oa[1])) <= hh[1] - margin;
        const bool lat2 = fabsf(fmaf(t, da[2], oa[2])) <= hh[2] - margin;
        const bool inside = t > 1e-4f && fabsf(da_sel) >= 0.05f && (a0 || lat0) && (a1 || lat1) && (a0 || a1 || lat2);
        if (inside) {
            const int face = (a0 ? 0 : (a1 ? 2 : 4)) + (da_sel > 0.0f ? 0 : 1);
            Hit fh{max_t, 0x7fffffff};
            const int s0 = kBoxFaceTris[face][0], s1 = kBoxFaceTris[face][1];
            tri_test(tp + 3 * s0, tri0 + s0, o, d, max_t, fh);
            tri_test(tp + 3 * s1, tri0 + s1, o, d, max_t, fh);
            if (fh.tri != 0x7fffffff) {
                if (fh.t < best.t || (fh.t == best.t && fh.tri < best.tri)) best = fh;
                return;
            }
        }
    }
    for (int s = 0; s < L; ++s) tri_test(tp + 3 * s, tri0 + s, o, d, max_t, best);
}

// closest hit of this lane's ray; all 32 lanes of the warp (one 8x4 tile, common origin o) must call it together
__device__ __forceinline__ Hit tile_closest_hit(const float* __restrict__ rec, int n_rec, const float* __restrict__ tris, int L, v3 o,
                                                v3 d, float max_t, int lane) {
    Hit best{max_t, 0x7fffffff};
    const TilePlanes tp = tile_planes(d, max_t);
    for (int base = 0; base < n_rec; base += 32) {
        const bool cand = (base + lane < n_rec) && tile_may_hit(tp, rec + (size_t)(base + lane) * kRecFloats);
        unsigned m = __ballot_sync(0xffffffffu, cand);
        while (m) {
            const int j = base + __ffs(m) - 1;
            m &= m - 1;
            record_object_test(rec + (size_t)j * kRecFloats, tris, L, o, d, max_t, best);
        }
    }
    return best;
}

// ---- a14: sphere vs triangle mesh (bit contract with oracle point_tri_dist2) ----------------
__device__ __forceinline__ float point_tri_dist2(v3 p, v3 a, v3 ab, v3 ac) {
    v3 ap = sub3(p, a);
    float d1 = dot3(ab, ap), d2 = dot3(ac, ap);
    if (d1 <= 0.0f && d2 <= 0.0f) return dot3(ap, ap);
    v3 b{a.x + ab.x, a.y + ab.y, a.z + ab.z};
    v3 bp = sub3(p, b);
    float d3 = dot3(ab, bp), d4 = dot3(ac, bp);
    if (d3 >= 0.0f && d4 <= d3) return dot3(bp, bp);
    float vc = fmaf(d1, d4, -(d3 * d2));
    if (vc <= 0.0f && d1 >= 0.0f && d3 <= 0.0f) {
        float v = d1 / (d1 - d3);
        v3 d = sub3(p, v3{fmaf(v, ab.x, a.x), fmaf(v, ab.y, a.y), fmaf(v, ab.z, a.z)});
        return dot3(d, d);
    }
    v3 c{a.x + ac.x, a.y + ac.y, a.z + ac.z};
    v3 cp = sub3(p, c);
    float d5 = dot3(ab, cp), d6 = dot3(ac, cp);
    if (d6 >= 0.0f && d5 <= d6) return dot3(cp, cp);
    float vb = fmaf(d5, d2, -(d1 * d6));
    if (vb <= 0.0f && d2 >= 0.0f && d6 <= 0.0f) {
        float w = d2 / (d2 - d6);
        v3 d = sub3(p, v3{fmaf(w, ac.x, a.x), fmaf(w, ac.y, a.y), fmaf(w, ac.z, a.z)});
        return dot3(d, d);
    }
    float va = fmaf(d3, d6, -(d5 * d4));
    if (va <= 0.0f && (d4 - d3) >= 0.0f && (d5 - d6) >= 0.0f) {
        float w = (d4 - d3) / ((d4 - d3) + (d5 - d6));
        v3 bc = sub3(c, b);
        v3 d = sub3(p, v3{fmaf(w, bc.x, b.x), fmaf(w, bc.y, b.y), fmaf(w, bc.z, b.z)});
        return dot3(d, d);
    }
    float denom = 1.0f / (va + vb + vc);
    float v = vb * denom, w = vc * denom;
    v3 d = sub3(p, v3{fmaf(w, ac.x, fmaf(v, ab.x, a.x)), fmaf(w, ac.y, fmaf(v, ab.y, a.y)), fmaf(w, ac.z, fmaf(v, ab.z, a.z))});
    return dot3(d, d);
}

// one mesh object: descend its BLAS with the same sphere/box test as the top level; min is order-independent, so the
// result is the oracle's min over the object's triangles within reach
__device__ __noinline__ float mesh_sphere_min(const AgxHp2Scene& sc, const MeshCtx& mc, int obj, v3 c, float search, float best) {
    const int m = sc.tmpl_mesh[mc.obj_template[obj]];
    const int2* topo = reinterpret_cast<const int2*>(sc.mesh_topo) + sc.mesh_node_offset[m];
    const float* nodes = mc.nodes + (size_t)mc.slot[2 * obj + 1] * kNodeFloats;
    const float4* tp = reinterpret_cast<const float4*>(mc.tris + (size_t)mc.slot[2 * obj] * kTriFloats);
    int stack[AGX_HP2_BLAS_MAX_DEPTH];
    int sp = 0, node = 0;
    while (true) {
        const float* nd = nodes + (size_t)node * kNodeFloats;
        float dx = fmaxf(fmaxf(nd[0] - c.x, c.x - nd[4]), 0.0f);
        float dy = fmaxf(fmaxf(nd[1] - c.y, c.y - nd[5]), 0.0f);
        float dz = fmaxf(fmaxf(nd[2] - c.z, c.z - nd[6]), 0.0f);
        float box_d2 = dx * dx + dy * dy + dz * dz;
        if (box_d2 <= fminf(best, search) * 1.0001f + 1e-6f) {  // culling only, as at the top level
            const int2 t = topo[node];
            if (t.y > 0) {
                for (int s = t.x; s < t.x + t.y; ++s) {
                    float4 a = tp[3 * s], b = tp[3 * s + 1], cc = tp[3 * s + 2];
                    best = fminf(best, point_tri_dist2(c, v3{a.x, a.y, a.z}, v3{b.x, b.y, b.z}, v3{cc.x, cc.y, cc.z}));
                }
            } else {
                stack[sp++] = t.x + 1;
                node = t.x;
                continue;
            }
        }
        if (sp == 0) break;
        node = stack[--sp];
    }
    return best;
}

// one thread per env: BVH descent with a sphere/AABB overlap test, exact min distance over the
// triangles of every leaf the sphere of the CURRENT best radius can reach
__global__ void __launch_bounds__(128)
hp2_collide_kernel(const __grid_constant__ AgxHp2Scene sc, const float* __restrict__ robot_pose, int stride, float radius,
                   uint8_t* __restrict__ crashes, float* __restrict__ min_dist) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= sc.num_envs) return;
    const int K = sc.num_objects, P = sc.leaves_pow2, L = sc.tris_per_object;
    const float* nodes = sc.nodes + (size_t)e * (2 * P - 1) * kNodeFloats;
    const int32_t* leaf = sc.leaf_object + (size_t)e * (P < 4 ? 4 : P);
    const float* tris = sc.tris + (size_t)e * K * L * kTriFloats;
    const float* rp = robot_pose + (size_t)e * stride;
    const v3 c{rp[0], rp[1], rp[2]};
    // search radius: exact min distance is only needed when min_dist is requested; otherwise the
    // collision radius bounds the search
    float best = 3.0e38f;
    const float r2 = radius * radius;
    const float search = min_dist ? 3.0e38f : r2;
    int stack[24];
    int sp = 0, node = 0;
    while (true) {
        const float* nd = nodes + (size_t)node * kNodeFloats;
        float dx = fmaxf(fmaxf(nd[0] - c.x, c.x - nd[4]), 0.0f);
        float dy = fmaxf(fmaxf(nd[1] - c.y, c.y - nd[5]), 0.0f);
        float dz = fmaxf(fmaxf(nd[2] - c.z, c.z - nd[6]), 0.0f);
        float box_d2 = dx * dx + dy * dy + dz * dz;
        float lim = fminf(best, search);
        bool reach = box_d2 <= lim * 1.0001f + 1e-6f;  // padded boxes + slack: culling only
        if (reach) {
            if (node >= P - 1) {
                int obj = leaf[node - (P - 1)];
                if (obj >= 0 && sc.num_meshes && sc.obj_mesh_slot[((size_t)e * K + obj) * 2] >= 0) {
                    best = mesh_sphere_min(sc, mesh_ctx(sc, e), obj, c, search, best);
                } else if (obj >= 0) {
                    const float4* tp = reinterpret_cast<const float4*>(tris + (size_t)obj * L * kTriFloats);
                    for (int s = 0; s < L; ++s) {
                        float4 a = tp[3 * s], b = tp[3 * s + 1], cc = tp[3 * s + 2];
                        if (b.x == 0.f && b.y == 0.f && b.z == 0.f && cc.x == 0.f && cc.y == 0.f && cc.z == 0.f) continue;  // padding slot
                        float d2 = point_tri_dist2(c, v3{a.x, a.y, a.z}, v3{b.x, b.y, b.z}, v3{cc.x, cc.y, cc.z});
                        best = fminf(best, d2);
                    }
                }
            } else {
                stack[sp++] = 2 * node + 2;
                node = 2 * node + 1;
                continue;
            }
        }
        if (sp == 0) break;
        node = stack[--sp];
    }
    if (best <= r2) crashes[e] = 1;
    if (min_dist) min_dist[e] = sqrtf(best);
}

// ---- contact mode (agx_hp2_contact): per object the closest point, then the solve of contact_core.cuh --------------------------
// point_tri_dist2's Voronoi regions, returning the closest point itself
__device__ __forceinline__ v3 closest_point_tri(v3 p, v3 a, v3 ab, v3 ac) {
    v3 ap = sub3(p, a);
    float d1 = dot3(ab, ap), d2 = dot3(ac, ap);
    if (d1 <= 0.0f && d2 <= 0.0f) return a;
    v3 b{a.x + ab.x, a.y + ab.y, a.z + ab.z};
    v3 bp = sub3(p, b);
    float d3 = dot3(ab, bp), d4 = dot3(ac, bp);
    if (d3 >= 0.0f && d4 <= d3) return b;
    float vc = fmaf(d1, d4, -(d3 * d2));
    if (vc <= 0.0f && d1 >= 0.0f && d3 <= 0.0f) {
        float v = d1 / (d1 - d3);
        return v3{fmaf(v, ab.x, a.x), fmaf(v, ab.y, a.y), fmaf(v, ab.z, a.z)};
    }
    v3 c{a.x + ac.x, a.y + ac.y, a.z + ac.z};
    v3 cp = sub3(p, c);
    float d5 = dot3(ab, cp), d6 = dot3(ac, cp);
    if (d6 >= 0.0f && d5 <= d6) return c;
    float vb = fmaf(d5, d2, -(d1 * d6));
    if (vb <= 0.0f && d2 >= 0.0f && d6 <= 0.0f) {
        float w = d2 / (d2 - d6);
        return v3{fmaf(w, ac.x, a.x), fmaf(w, ac.y, a.y), fmaf(w, ac.z, a.z)};
    }
    float va = fmaf(d3, d6, -(d5 * d4));
    if (va <= 0.0f && (d4 - d3) >= 0.0f && (d5 - d6) >= 0.0f) {
        float w = (d4 - d3) / ((d4 - d3) + (d5 - d6));
        v3 bc = sub3(c, b);
        return v3{fmaf(w, bc.x, b.x), fmaf(w, bc.y, b.y), fmaf(w, bc.z, b.z)};
    }
    float denom = 1.0f / (va + vb + vc);
    float v = vb * denom, w = vc * denom;
    return v3{fmaf(w, ac.x, fmaf(v, ab.x, a.x)), fmaf(w, ac.y, fmaf(v, ab.y, a.y)), fmaf(w, ac.z, fmaf(v, ab.z, a.z))};
}

// the closest triangle of one object: squared distance, closest point, the triangle's slab (its face normal when d2 == 0)
struct ObjClosest {
    float d2;
    v3 q;
    const float4* tri;
};
__device__ __forceinline__ void tri_closest(v3 c, const float4* tp, ObjClosest& best) {
    const float4 a = tp[0], b = tp[1], cc = tp[2];
    const v3 q = closest_point_tri(c, v3{a.x, a.y, a.z}, v3{b.x, b.y, b.z}, v3{cc.x, cc.y, cc.z});
    const v3 d = sub3(c, q);
    const float d2 = dot3(d, d);
    if (d2 < best.d2) best = ObjClosest{d2, q, tp};
}

// one mesh object: the BLAS descent of mesh_sphere_min, keeping the closest point
__device__ __noinline__ void mesh_closest(const AgxHp2Scene& sc, const MeshCtx& mc, int obj, v3 c, float search, ObjClosest& best) {
    const int m = sc.tmpl_mesh[mc.obj_template[obj]];
    const int2* topo = reinterpret_cast<const int2*>(sc.mesh_topo) + sc.mesh_node_offset[m];
    const float* nodes = mc.nodes + (size_t)mc.slot[2 * obj + 1] * kNodeFloats;
    const float4* tp = reinterpret_cast<const float4*>(mc.tris + (size_t)mc.slot[2 * obj] * kTriFloats);
    int stack[AGX_HP2_BLAS_MAX_DEPTH];
    int sp = 0, node = 0;
    while (true) {
        const float* nd = nodes + (size_t)node * kNodeFloats;
        float dx = fmaxf(fmaxf(nd[0] - c.x, c.x - nd[4]), 0.0f);
        float dy = fmaxf(fmaxf(nd[1] - c.y, c.y - nd[5]), 0.0f);
        float dz = fmaxf(fmaxf(nd[2] - c.z, c.z - nd[6]), 0.0f);
        float box_d2 = dx * dx + dy * dy + dz * dz;
        if (box_d2 <= fminf(best.d2, search) * 1.0001f + 1e-6f) {  // culling only
            const int2 t = topo[node];
            if (t.y > 0) {
                for (int s = t.x; s < t.x + t.y; ++s) tri_closest(c, tp + 3 * s, best);
            } else {
                stack[sp++] = t.x + 1;
                node = t.x;
                continue;
            }
        }
        if (sp == 0) break;
        node = stack[--sp];
    }
}

// one thread per env: every object within reach (radius + contact_offset) gives its closest point, the ground plane one more;
// the AGX_CONTACT_MAX nearest go to the solve.  sc.num_objects == 0: no scene.
__global__ void __launch_bounds__(128)
hp2_contact_kernel(const __grid_constant__ AgxHp2Scene sc, const __grid_constant__ AgxContactParams P, int num_envs,
                   float* __restrict__ root_state, int stride, float* __restrict__ force, uint8_t* __restrict__ crashes,
                   int32_t* __restrict__ contact_obj) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= num_envs) return;
    float* rs = root_state + (size_t)e * stride;
    const v3 c{rs[0], rs[1], rs[2]};
    const float reach = P.radius + P.contact_offset;
    const float search = reach * reach;
    agx::ContactPt cp[AGX_CONTACT_MAX];
    float key[AGX_CONTACT_MAX];
    int id[AGX_CONTACT_MAX];
    int n = 0;
    const int K = sc.num_objects;
    if (K > 0) {
        const int P2 = sc.leaves_pow2, L = sc.tris_per_object;
        const float* nodes = sc.nodes + (size_t)e * (2 * P2 - 1) * kNodeFloats;
        const int32_t* leaf = sc.leaf_object + (size_t)e * (P2 < 4 ? 4 : P2);
        const float* tris = sc.tris + (size_t)e * K * L * kTriFloats;
        int stack[24];
        int sp = 0, node = 0;
        while (true) {
            const float* nd = nodes + (size_t)node * kNodeFloats;
            float dx = fmaxf(fmaxf(nd[0] - c.x, c.x - nd[4]), 0.0f);
            float dy = fmaxf(fmaxf(nd[1] - c.y, c.y - nd[5]), 0.0f);
            float dz = fmaxf(fmaxf(nd[2] - c.z, c.z - nd[6]), 0.0f);
            float box_d2 = dx * dx + dy * dy + dz * dz;
            if (box_d2 <= search * 1.0001f + 1e-6f) {  // padded boxes + slack: culling only
                if (node >= P2 - 1) {
                    const int obj = leaf[node - (P2 - 1)];
                    ObjClosest best{3.0e38f, v3{0.0f, 0.0f, 0.0f}, nullptr};
                    if (obj >= 0 && sc.num_meshes && sc.obj_mesh_slot[((size_t)e * K + obj) * 2] >= 0) {
                        mesh_closest(sc, mesh_ctx(sc, e), obj, c, search, best);
                    } else if (obj >= 0) {
                        const float4* tp = reinterpret_cast<const float4*>(tris + (size_t)obj * L * kTriFloats);
                        for (int s = 0; s < L; ++s) {
                            const float4 b = tp[3 * s + 1], cc = tp[3 * s + 2];
                            if (b.x == 0.f && b.y == 0.f && b.z == 0.f && cc.x == 0.f && cc.y == 0.f && cc.z == 0.f) continue;  // padding
                            tri_closest(c, tp + 3 * s, best);
                        }
                    }
                    if (best.d2 <= search) {
                        const float dist = sqrtf(best.d2);
                        v3 nv;
                        if (dist > 0.0f) {
                            const v3 d = sub3(c, best.q);
                            nv = v3{d.x / dist, d.y / dist, d.z / dist};
                        } else {  // the centre lies on the surface: the triangle's face normal
                            const float4 b = best.tri[1], cc = best.tri[2];
                            nv = normalize3(cross3(v3{b.x, b.y, b.z}, v3{cc.x, cc.y, cc.z}));
                        }
                        const agx::ContactPt pt{{best.q.x, best.q.y, best.q.z}, {nv.x, nv.y, nv.z}, P.radius - dist};
                        n = agx::contact_insert(cp, key, id, n, pt, dist, obj);
                    }
                } else {
                    stack[sp++] = 2 * node + 2;
                    node = 2 * node + 1;
                    continue;
                }
            }
            if (sp == 0) break;
            node = stack[--sp];
        }
    }
    if (P.ground_plane && c.z <= reach) {
        const agx::ContactPt pt{{c.x, c.y, 0.0f}, {0.0f, 0.0f, 1.0f}, P.radius - c.z};
        n = agx::contact_insert(cp, key, id, n, pt, c.z, K);
    }
    if (contact_obj)
        for (int i = 0; i < AGX_CONTACT_MAX; ++i) contact_obj[(size_t)e * AGX_CONTACT_MAX + i] = i < n ? id[i] : -1;
    float* f = force + (size_t)e * 3;
    if (n == 0) {
        f[0] = f[1] = f[2] = 0.0f;
        return;
    }
    agx::contact_env(P, rs, cp, n, f, crashes + e);
}

// hp2_contact_kernel's contact search for one env (centre c), as a function: the nearest contacts in cp / key / id, their count
// returned.  hp2_contact_kernel keeps its inline copy so that its machine code stays as it was verified: inlining this function
// there lays out its stack frame differently.
__device__ __forceinline__ int contact_search(const AgxHp2Scene& sc, const AgxContactParams& P, int e, v3 c, agx::ContactPt* cp, float* key,
                                              int* id) {
    const float reach = P.radius + P.contact_offset;
    const float search = reach * reach;
    int n = 0;
    const int K = sc.num_objects;
    if (K > 0) {
        const int P2 = sc.leaves_pow2, L = sc.tris_per_object;
        const float* nodes = sc.nodes + (size_t)e * (2 * P2 - 1) * kNodeFloats;
        const int32_t* leaf = sc.leaf_object + (size_t)e * (P2 < 4 ? 4 : P2);
        const float* tris = sc.tris + (size_t)e * K * L * kTriFloats;
        int stack[24];
        int sp = 0, node = 0;
        while (true) {
            const float* nd = nodes + (size_t)node * kNodeFloats;
            float dx = fmaxf(fmaxf(nd[0] - c.x, c.x - nd[4]), 0.0f);
            float dy = fmaxf(fmaxf(nd[1] - c.y, c.y - nd[5]), 0.0f);
            float dz = fmaxf(fmaxf(nd[2] - c.z, c.z - nd[6]), 0.0f);
            float box_d2 = dx * dx + dy * dy + dz * dz;
            if (box_d2 <= search * 1.0001f + 1e-6f) {  // padded boxes + slack: culling only
                if (node >= P2 - 1) {
                    const int obj = leaf[node - (P2 - 1)];
                    ObjClosest best{3.0e38f, v3{0.0f, 0.0f, 0.0f}, nullptr};
                    if (obj >= 0 && sc.num_meshes && sc.obj_mesh_slot[((size_t)e * K + obj) * 2] >= 0) {
                        mesh_closest(sc, mesh_ctx(sc, e), obj, c, search, best);
                    } else if (obj >= 0) {
                        const float4* tp = reinterpret_cast<const float4*>(tris + (size_t)obj * L * kTriFloats);
                        for (int s = 0; s < L; ++s) {
                            const float4 b = tp[3 * s + 1], cc = tp[3 * s + 2];
                            if (b.x == 0.f && b.y == 0.f && b.z == 0.f && cc.x == 0.f && cc.y == 0.f && cc.z == 0.f) continue;  // padding
                            tri_closest(c, tp + 3 * s, best);
                        }
                    }
                    if (best.d2 <= search) {
                        const float dist = sqrtf(best.d2);
                        v3 nv;
                        if (dist > 0.0f) {
                            const v3 d = sub3(c, best.q);
                            nv = v3{d.x / dist, d.y / dist, d.z / dist};
                        } else {  // the centre lies on the surface: the triangle's face normal
                            const float4 b = best.tri[1], cc = best.tri[2];
                            nv = normalize3(cross3(v3{b.x, b.y, b.z}, v3{cc.x, cc.y, cc.z}));
                        }
                        const agx::ContactPt pt{{best.q.x, best.q.y, best.q.z}, {nv.x, nv.y, nv.z}, P.radius - dist};
                        n = agx::contact_insert(cp, key, id, n, pt, dist, obj);
                    }
                } else {
                    stack[sp++] = 2 * node + 2;
                    node = 2 * node + 1;
                    continue;
                }
            }
            if (sp == 0) break;
            node = stack[--sp];
        }
    }
    if (P.ground_plane && c.z <= reach) {
        const agx::ContactPt pt{{c.x, c.y, 0.0f}, {0.0f, 0.0f, 1.0f}, P.radius - c.z};
        n = agx::contact_insert(cp, key, id, n, pt, c.z, K);
    }
    return n;
}

// hp2_contact_kernel with moving obstacles: each kept object contact also gets its obstacle's velocity at the contact point, from
// the row of the asset that owns the object (mo.obj_asset, in range by the caller's contract); the ground's is 0
__global__ void __launch_bounds__(128)
hp2_contact_moving_kernel(const __grid_constant__ AgxHp2Scene sc, const __grid_constant__ AgxContactParams P,
                          const __grid_constant__ AgxContactMotion mo, int num_envs, float* __restrict__ root_state, int stride,
                          float* __restrict__ force, uint8_t* __restrict__ crashes, int32_t* __restrict__ contact_obj) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= num_envs) return;
    float* rs = root_state + (size_t)e * stride;
    agx::ContactPt cp[AGX_CONTACT_MAX];
    float key[AGX_CONTACT_MAX];
    int id[AGX_CONTACT_MAX];
    const int n = contact_search(sc, P, e, v3{rs[0], rs[1], rs[2]}, cp, key, id);
    if (contact_obj)
        for (int i = 0; i < AGX_CONTACT_MAX; ++i) contact_obj[(size_t)e * AGX_CONTACT_MAX + i] = i < n ? id[i] : -1;
    float* f = force + (size_t)e * 3;
    if (n == 0) {
        f[0] = f[1] = f[2] = 0.0f;
        return;
    }
    const int K = sc.num_objects;
    float u[AGX_CONTACT_MAX][3];
    for (int i = 0; i < n; ++i) {
        if (id[i] < K) {
            const int a = mo.obj_asset[(size_t)e * K + id[i]];
            agx::obstacle_point_vel(mo.asset_state + ((size_t)e * mo.num_assets + a) * mo.asset_stride, cp[i].p, u[i]);
        } else {
            u[i][0] = u[i][1] = u[i][2] = 0.0f;
        }
    }
    agx::contact_env<true>(P, rs, cp, n, f, crashes + e, u);
}

// hp2_contact_moving_kernel with dynamic obstacles: the assets of the kept object contacts become the bodies of the two-body solve
// (at most AGX_CONTACT_MAX per env, one per distinct asset, in the order of their first contact), loaded from their rows and mass
// entries, solved with the robot, and the free ones written back to their rows.  Only this env's thread touches this env's rows.
__global__ void __launch_bounds__(128)
hp2_contact_dynamic_kernel(const __grid_constant__ AgxHp2Scene sc, const __grid_constant__ AgxContactParams P,
                           const __grid_constant__ AgxContactMotion mo, float* __restrict__ asset_state,
                           const AgxObstacleMass* __restrict__ mass, int num_envs, float* __restrict__ root_state, int stride,
                           float* __restrict__ force, uint8_t* __restrict__ crashes, int32_t* __restrict__ contact_obj) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= num_envs) return;
    float* rs = root_state + (size_t)e * stride;
    agx::ContactPt cp[AGX_CONTACT_MAX];
    float key[AGX_CONTACT_MAX];
    int id[AGX_CONTACT_MAX];
    const int n = contact_search(sc, P, e, v3{rs[0], rs[1], rs[2]}, cp, key, id);
    if (contact_obj)
        for (int i = 0; i < AGX_CONTACT_MAX; ++i) contact_obj[(size_t)e * AGX_CONTACT_MAX + i] = i < n ? id[i] : -1;
    float* f = force + (size_t)e * 3;
    if (n == 0) {
        f[0] = f[1] = f[2] = 0.0f;
        return;
    }
    const int K = sc.num_objects, A = mo.num_assets;
    agx::ContactBody B[AGX_CONTACT_MAX];
    float* rows[AGX_CONTACT_MAX];
    int body[AGX_CONTACT_MAX];
    const int nb = agx::contact_bodies_gather(id, n, K, mo.obj_asset + (size_t)e * K, asset_state + (size_t)e * A * mo.asset_stride,
                                              mo.asset_stride, mass + (size_t)e * A, B, rows, body);
    agx::contact_env_dynamic(P, rs, cp, n, f, crashes + e, body, B, nb, rows);
}

__device__ __forceinline__ float range_epilogue(const AgxHp2Sensor& s, float px) {
    // warp_sensor.py:216-225: two sequential masked assignments, then the division
    if (px > s.max_range) px = s.far_out_of_range_value;
    if (px < s.min_range) px = s.near_out_of_range_value;
    if (s.normalize_range && !s.pointcloud_in_world_frame) px = px / s.max_range;
    return px;
}

constexpr int kCastThreads = 256;

// 4 CTAs of 256 threads per SM (<= 64 registers): the kernel is latency bound, 32 resident warps per SM
// measured 2.0x faster than 16 (tools/dbg/build_variant.sh) despite ~200 B of spills
#ifndef AGX_CAST_MIN_BLOCKS
#define AGX_CAST_MIN_BLOCKS 4
#endif
// MESH: scene with mesh objects (num_meshes > 0; per-ray traversal only, TILE = false)
template <bool SMEM, bool TILE = false, bool MESH = false>
__global__ void __launch_bounds__(kCastThreads, AGX_CAST_MIN_BLOCKS)
hp2_cast_kernel(const __grid_constant__ AgxHp2Scene sc, const __grid_constant__ AgxHp2Sensor sn, int rows_per_item,
                int items_per_image, long long n_items, int rec_cap) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ __align__(8) uint64_t s_bar;
    __shared__ int s_nrec;
    const int K = sc.num_objects, P = sc.leaves_pow2, L = sc.tris_per_object;
    const int W = sn.width, H = sn.height, S = sn.num_sensors;
    const uint32_t node_bytes = (uint32_t)((2 * P - 1) * kNodeFloats * 4);
    const int leaf_stride = P < 4 ? 4 : P;  // 16-byte granularity of cp.async.bulk
    const uint32_t leaf_bytes = (uint32_t)(leaf_stride * 4);
    const uint32_t tri_bytes = (uint32_t)((size_t)K * L * kTriFloats * 4);
    float* s_nodes = reinterpret_cast<float*>(smem_raw);
    int32_t* s_leaf = reinterpret_cast<int32_t*>(smem_raw + ((node_bytes + 15u) & ~15u));
    float* s_tris = reinterpret_cast<float*>(reinterpret_cast<unsigned char*>(s_leaf) + ((leaf_bytes + 15u) & ~15u));
    const uint32_t obb_bytes = sc.obb ? (uint32_t)((size_t)K * kObbFloats * 4) : 0u;
    float* s_obb = reinterpret_cast<float*>(reinterpret_cast<unsigned char*>(s_tris) + tri_bytes);
    // TILE only: object records behind the staged scene, or (scene too large to stage: <false, true>) at the start of the buffer
    float* s_rec = SMEM ? reinterpret_cast<float*>(reinterpret_cast<unsigned char*>(s_obb) + ((obb_bytes + 15u) & ~15u)) : reinterpret_cast<float*>(smem_raw);
    if (SMEM && threadIdx.x == 0) {
        mbar_init(&s_bar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    uint32_t parity = 0;
    int staged_env = -1;
    const q4 qf{sn.frame_quat[0], sn.frame_quat[1], sn.frame_quat[2], sn.frame_quat[3]};

    for (long long item = blockIdx.x; item < n_items; item += gridDim.x) {
        const int rb = (int)(item % items_per_image);
        const long long es = item / items_per_image;
        const int c = (int)(es % S);
        const int e = (int)(es / S);
        const float* g_nodes = sc.nodes + (size_t)e * (2 * P - 1) * kNodeFloats;
        const int32_t* g_leaf = sc.leaf_object + (size_t)e * leaf_stride;
        const float* g_tris = sc.tris + (size_t)e * K * L * kTriFloats;
        const float* g_obb = sc.obb ? sc.obb + (size_t)e * K * kObbFloats : nullptr;
        const float* nodes = g_nodes;
        const int32_t* leaf = g_leaf;
        const float* tris = g_tris;
        const float* obb = g_obb;
        MeshCtx mc{};
        if constexpr (MESH) mc = mesh_ctx(sc, e);
        bool fresh_scene = false;  // uniform: this item staged a new scene (its leading barrier also retired the previous item's records)
        if (SMEM) {
            if (e != staged_env) {
                __syncthreads();  // everyone is done with the previous scene (and with the previous item's records)
                if (threadIdx.x == 0) {
                    // record count of the new item: written before the mbarrier arrive (release) below, read by the others after their
                    // mbar_wait (acquire) -- no CTA barrier of its own (ncu r1/r2: `barrier` was the top stall of this kernel)
                    if (TILE) s_nrec = 0;
                    // order prior generic-proxy smem reads before the async-proxy writes
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                    mbar_expect_tx(&s_bar, node_bytes + leaf_bytes + tri_bytes + obb_bytes);
                    tma_bulk_g2s(s_nodes, g_nodes, node_bytes, &s_bar);
                    tma_bulk_g2s(s_leaf, g_leaf, leaf_bytes, &s_bar);
                    tma_bulk_g2s(s_tris, g_tris, tri_bytes, &s_bar);
                    if (obb_bytes) tma_bulk_g2s(s_obb, g_obb, obb_bytes, &s_bar);
                }
                mbar_wait(&s_bar, parity);
                parity ^= 1u;
                staged_env = e;
                fresh_scene = true;
            }
            nodes = s_nodes;
            leaf = s_leaf;
            tris = s_tris;
            if (obb_bytes) obb = s_obb;
        }
        // ---- sensor pose: warp_sensor.py:180-187 ------------------------------------------------
        const float* rp = sn.robot_pose + (size_t)e * sn.robot_pose_stride;
        const float* m = sn.mount + ((size_t)e * S + c) * 7;
        q4 rq{rp[3], rp[4], rp[5], rp[6]};
        v3 sp = quat_apply(rq, v3{m[0], m[1], m[2]});
        sp.x += rp[0]; sp.y += rp[1]; sp.z += rp[2];
        q4 sq = quat_mul(rq, quat_mul(q4{m[3], m[4], m[5], m[6]}, qf));
        v3 rd_p{0.f, 0.f, 0.f};
        const bool is_cam = sn.kind == AGX_SENSOR_CAMERA || sn.kind == AGX_SENSOR_STEREO_CAMERA || sn.kind == AGX_SENSOR_NORMAL_FACEID_CAMERA;
        const bool is_normal = sn.kind == AGX_SENSOR_NORMAL_FACEID_CAMERA || sn.kind == AGX_SENSOR_NORMAL_FACEID_LIDAR;
        const bool norm_uv = sn.return_pointcloud || sn.kind == AGX_SENSOR_NORMAL_FACEID_CAMERA;
        v3 stereo_pos = sp;
        if (sn.kind == AGX_SENSOR_STEREO_CAMERA) {  // warp_stereo_camera_kernels.py:180-181
            v3 ro = quat_rotate(sq, v3{-sn.baseline, 0.0f, 0.0f});
            stereo_pos = v3{sp.x + ro.x, sp.y + ro.y, sp.z + ro.z};
        }
        if (is_cam) {
            v3 uvp = kinv_mul(sn.kinv, v3{(float)sn.c_x, (float)sn.c_y, 1.0f});
            if (norm_uv) uvp = normalize3(uvp);
            rd_p = normalize3(quat_rotate(sq, uvp));
        }
        const int y0 = rb * rows_per_item;
        const int y1 = min(H, y0 + rows_per_item);
        // warp <-> 8x4 pixel tile: neighbouring rays stay in one warp (coherent traversal, SIMT efficiency)
        const int tiles_x = (W + 7) >> 3, tiles_y = (y1 - y0 + 3) >> 2;
        const int lane = threadIdx.x & 31, lx = lane & 7, ly = lane >> 3;
        // Tile path.  <true, true>: scene staged in shared memory (<= 128 leaf slots, every shipped environment).  <false, true>: scene
        // too large to stage (BASELINE configs[2]: 1024 boxes = 590 KB): the records of the objects that survive the work item's
        // frustum (a 4096-ray row block: a few percent of a cluttered scene) still fit shared memory, the per-tile culling and the
        // uniform candidate loop are the same, only the candidates' triangle slabs come from L2 -- no per-ray BVH walk with its
        // divergent stack.  If more objects survive than there are record slots (LiDAR row blocks span the full azimuth), this
        // work item walks the BVH per ray as before.
        constexpr bool tile_path = TILE;
        if constexpr (tile_path) {  // per-item object records (depend on the sensor origin)
            if (!fresh_scene) {     // same scene as the previous item (row blocks of a large image), or no staging at all
                __syncthreads();    // previous item's records are no longer read
                if (threadIdx.x == 0) s_nrec = 0;
                __syncthreads();
            }
            v3 fr[4];
            bool have_frustum = false;
            float item_far = sn.far_plane;
            if (is_cam) {  // corner rays of this item's pixel block, same arithmetic as the per-pixel rays below
                const float xs[2] = {0.0f, (float)(W - 1)}, ys[2] = {(float)(rb * rows_per_item), (float)(min(H, rb * rows_per_item + rows_per_item) - 1)};
                v3 cd[4];
                float min_mult = 1.0f;
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    v3 cuv = kinv_mul(sn.kinv, v3{xs[(k == 1 || k == 2) ? 1 : 0], ys[k >> 1], 1.0f});
                    if (norm_uv) cuv = normalize3(cuv);
                    cd[k] = normalize3(quat_rotate(sq, cuv));
                    min_mult = fminf(min_mult, dot3(cd[k], rd_p));
                }
                // the planes are only meaningful for a pyramid narrower than a half space
                const v3 dcs{cd[0].x + cd[1].x + cd[2].x + cd[3].x, cd[0].y + cd[1].y + cd[2].y + cd[3].y, cd[0].z + cd[1].z + cd[2].z + cd[3].z};
                have_frustum = min_mult > 0.2f;
                fr[0] = cross3(cd[0], cd[1]); fr[1] = cross3(cd[1], cd[2]); fr[2] = cross3(cd[2], cd[3]); fr[3] = cross3(cd[3], cd[0]);
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    if (dot3(fr[k], dcs) < 0.0f) fr[k] = v3{-fr[k].x, -fr[k].y, -fr[k].z};
                    // every corner ray must be on the inner side of every plane, else do not trust the pyramid
                    for (int j = 0; j < 4; ++j)
                        if (dot3(fr[k], cd[j]) < -1e-5f * sqrtf(dot3(fr[k], fr[k]))) have_frustum = false;
                }
                if (sn.kind != AGX_SENSOR_NORMAL_FACEID_CAMERA && !sn.return_pointcloud && sn.calculate_depth && min_mult > 0.2f)
                    item_far = sn.far_plane / min_mult;  // largest per-pixel max_t of the block is at a corner
                else if (sn.kind != AGX_SENSOR_NORMAL_FACEID_CAMERA && !sn.return_pointcloud && sn.calculate_depth)
                    item_far = FLT_MAX;
            }
            build_records(nodes, leaf, obb, P, sp, have_frustum ? fr : nullptr, item_far, s_rec, &s_nrec, rec_cap);
            __syncthreads();
        }
        const int n_rec = tile_path ? s_nrec : 0;
        const bool rec_overflow = tile_path && n_rec > rec_cap;
        for (int tix = threadIdx.x >> 5; tix < tiles_x * tiles_y; tix += kCastThreads / 32) {
            int x = (tix % tiles_x) * 8 + lx, y = y0 + (tix / tiles_x) * 4 + ly;
            const bool in_image = x < W && y < y1;
            if (!tile_path && !in_image) continue;
            x = min(x, W - 1);  // tile path: border lanes shadow the nearest pixel (they take part in the
            y = min(y, y1 - 1); // warp-wide culling) and skip the stores
            v3 uv, rd;
            float mult = 1.0f, max_t = sn.far_plane;
            if (is_cam) {  // warp_camera_kernels.py:186-221
                uv = kinv_mul(sn.kinv, v3{(float)x, (float)y, 1.0f});
                if (norm_uv) uv = normalize3(uv);
                rd = normalize3(quat_rotate(sq, uv));
                if (sn.kind != AGX_SENSOR_NORMAL_FACEID_CAMERA && !sn.return_pointcloud && sn.calculate_depth) {
                    mult = dot3(rd, rd_p);
                    max_t = sn.far_plane / mult;
                }
            } else {  // warp_lidar_kernels.py:24-33
                const float* rt = sn.ray_table + ((size_t)y * W + x) * 3;
                uv = normalize3(v3{rt[0], rt[1], rt[2]});
                rd = normalize3(quat_rotate(sq, uv));
            }
            typename std::conditional<MESH, MeshHit, Hit>::type h;
            if constexpr (tile_path) {
                if (!rec_overflow) h = tile_closest_hit(s_rec, n_rec, tris, L, sp, rd, max_t, lane);
                else h = traverse<SMEM, MESH>(nodes, leaf, tris, obb, P, L, sp, rd, max_t, &sc, &mc);
                if (!in_image) continue;
            } else {
                h = traverse<SMEM, MESH>(nodes, leaf, tris, obb, P, L, sp, rd, max_t, &sc, &mc);
            }
            float dist = AGX_NO_HIT_RAY_VAL;
            int segv = AGX_NO_HIT_SEG_VAL;
            const bool hit = h.tri != 0x7fffffff;
            const size_t pix = (((size_t)e * S + c) * H + y) * W + x;
            if (is_normal) {  // warp_camera_kernels.py:70-121, warp_lidar_kernels.py:90-126
                v3 o{0.f, 0.f, 0.f};
                int face = -1;
                if (hit) {
                    const float4* tp = reinterpret_cast<const float4*>(hit_slab<MESH>(h, tris, mc));
                    float4 b = tp[1], cc = tp[2];
                    v3 nrm = normalize3(cross3(v3{b.x, b.y, b.z}, v3{cc.x, cc.y, cc.z}));
                    if (sn.normal_in_world_frame) o = nrm;
                    else if (sn.kind == AGX_SENSOR_NORMAL_FACEID_CAMERA)
                        o = v3{dot3(nrm, rd_p), dot3(nrm, cross3(rd_p, v3{0.f, 0.f, 1.f})), dot3(nrm, cross3(rd_p, v3{0.f, 1.f, 0.f}))};
                    else
                        o = normalize3(quat_rotate(q4{-sq.x, -sq.y, -sq.z, sq.w}, nrm));
                    if constexpr (MESH) {
                        face = h.tri;
                    } else {
                        int obj = h.tri / L;
                        face = (sc.face_offset ? sc.face_offset[(size_t)e * K + obj] : obj * L) + (h.tri - obj * L);
                    }
                }
                sn.pixels[pix * 3 + 0] = o.x; sn.pixels[pix * 3 + 1] = o.y; sn.pixels[pix * 3 + 2] = o.z;
                if (sn.seg_pixels) sn.seg_pixels[pix] = face;
                continue;
            }
            if (sn.kind == AGX_SENSOR_STEREO_CAMERA) {  // warp_stereo_camera_kernels.py:205-222
                dist = -1.0f;  // INVALID_PIXEL_VAL
                v3 ep;
                if (hit) ep = v3{fmaf(rd.x * h.t, 0.999f, sp.x), fmaf(rd.y * h.t, 0.999f, sp.y), fmaf(rd.z * h.t, 0.999f, sp.z)};
                else ep = v3{sp.x + (rd.x * sn.far_plane) / mult, sp.y + (rd.y * sn.far_plane) / mult, sp.z + (rd.z * sn.far_plane) / mult};
                v3 dv = sub3(stereo_pos, ep);
                float dl = sqrtf(dot3(dv, dv));
                Hit h2 = traverse<SMEM, MESH>(nodes, leaf, tris, obb, P, L, ep, normalize3(dv), dl, &sc, &mc);
                const bool visible = h2.tri == 0x7fffffff;
                if (hit && visible) {
                    dist = h.t * mult;
                    segv = __float_as_int((hit_slab<MESH>(h, tris, mc))[3]);
                } else if (!hit && visible) {
                    dist = AGX_NO_HIT_RAY_VAL;
                }
                sn.pixels[pix] = sn.fuse_epilogue ? range_epilogue(sn, dist) : dist;
                if (sn.seg_pixels) sn.seg_pixels[pix] = segv;
                continue;
            }
            if (hit) {
                dist = mult * h.t;
                segv = __float_as_int((hit_slab<MESH>(h, tris, mc))[3]);
            }
            if (sn.return_pointcloud) {
                v3 p;
                if (sn.pointcloud_in_world_frame) p = v3{fmaf(dist, rd.x, sp.x), fmaf(dist, rd.y, sp.y), fmaf(dist, rd.z, sp.z)};
                else p = v3{dist * uv.x, dist * uv.y, dist * uv.z};
                if (sn.fuse_epilogue && !sn.pointcloud_in_world_frame) {  // warp_sensor.py:203-215
                    float nrm = sqrtf(dot3(p, p));
                    if (nrm > sn.max_range) p = v3{sn.far_out_of_range_value, sn.far_out_of_range_value, sn.far_out_of_range_value};
                    nrm = sqrtf(dot3(p, p));
                    if (nrm < sn.min_range) p = v3{sn.near_out_of_range_value, sn.near_out_of_range_value, sn.near_out_of_range_value};
                    if (sn.normalize_range) p = v3{p.x / sn.max_range, p.y / sn.max_range, p.z / sn.max_range};
                }
                sn.pixels[pix * 3 + 0] = p.x; sn.pixels[pix * 3 + 1] = p.y; sn.pixels[pix * 3 + 2] = p.z;
            } else {
                sn.pixels[pix] = sn.fuse_epilogue ? range_epilogue(sn, dist) : dist;
            }
            if (sn.seg_pixels) sn.seg_pixels[pix] = segv;
        }
    }
}

inline int next_pow2(int v) {
    int p = 1;
    while (p < v) p <<= 1;
    return p;
}
inline size_t record_smem_bytes(int K) { return (size_t)K * kRecFloats * 4 + 16; }
inline size_t scene_smem_bytes(int K, int P, int L, bool with_obb) {
    size_t nb = ((size_t)(2 * P - 1) * kNodeFloats * 4 + 15) & ~(size_t)15;
    size_t lb = (size_t)(P < 4 ? 4 : P) * 4;
    return nb + lb + (size_t)K * L * kTriFloats * 4 + (with_obb ? (size_t)K * kObbFloats * 4 : 0);
}

int validate_scene(const AgxHp2Scene* sc) {
    if (!sc) return agx_set_error(AGX_E_NULL, "scene is NULL");
    if (sc->num_objects < 1 || sc->num_objects > AGX_HP2_MAX_OBJECTS)
        return agx_set_error(AGX_E_INVALID, "num_objects must be in [1, %d]", AGX_HP2_MAX_OBJECTS);
    if (sc->leaves_pow2 != next_pow2(sc->num_objects)) return agx_set_error(AGX_E_INVALID, "leaves_pow2 must be the next power of two >= num_objects");
    if (sc->tris_per_object < 1 || sc->tris_per_object > 64) return agx_set_error(AGX_E_INVALID, "tris_per_object must be in [1, 64]");
    if (!sc->tris || !sc->nodes || !sc->leaf_object) return agx_set_error(AGX_E_NULL, "scene storage (tris/nodes/leaf_object) is NULL");
    if ((sc->tmpl_obb == nullptr) != (sc->obb == nullptr)) return agx_set_error(AGX_E_INVALID, "tmpl_obb and obb must be given together");
    if ((uintptr_t)sc->obb & 15) return agx_set_error(AGX_E_INVALID, "obb storage must be 16-byte aligned");
    if (((uintptr_t)sc->tris | (uintptr_t)sc->nodes | (uintptr_t)sc->leaf_object) & 15) return agx_set_error(AGX_E_INVALID, "scene storage must be 16-byte aligned");
    if (sc->num_meshes < 0 || sc->num_meshes > sc->num_templates) return agx_set_error(AGX_E_INVALID, "num_meshes must be in [0, num_templates]");
    if (sc->num_meshes) {
        if (!sc->tmpl_mesh || !sc->mesh_tri_offset || !sc->mesh_tris || !sc->mesh_tri_index || !sc->mesh_seg || !sc->mesh_node_offset ||
            !sc->mesh_topo || !sc->mesh_levels || !sc->obj_mesh_slot || !sc->mesh_world_tris || !sc->mesh_world_nodes)
            return agx_set_error(AGX_E_NULL, "mesh tables / storage are NULL");
        if (!sc->face_offset) return agx_set_error(AGX_E_NULL, "a scene with mesh objects needs face_offset");
        if (sc->mesh_tris_per_env < 1 || sc->mesh_nodes_per_env < 1)
            return agx_set_error(AGX_E_INVALID, "mesh_tris_per_env and mesh_nodes_per_env must be positive");
        if (((uintptr_t)sc->mesh_world_tris | (uintptr_t)sc->mesh_world_nodes | (uintptr_t)sc->mesh_topo) & 15)
            return agx_set_error(AGX_E_INVALID, "mesh storage must be 16-byte aligned");
    }
    return AGX_OK;
}

// the argument checks of both contact entry points; *launch = false: valid, nothing to do (no envs)
int contact_check(const AgxHp2Scene* sc, int num_envs, const AgxContactParams* p, const float* root_state, int root_state_stride,
                  const float* contact_force, const uint8_t* crashes, bool* launch) {
    *launch = false;
    if (sc) {
        int rc = validate_scene(sc);
        if (rc) return rc;
        if (sc->num_envs != num_envs) return agx_set_error(AGX_E_INVALID, "num_envs %d != scene num_envs %d", num_envs, sc->num_envs);
    }
    if (!p) return agx_set_error(AGX_E_NULL, "params is NULL");
    if (num_envs < 0) return agx_set_error(AGX_E_INVALID, "num_envs < 0");
    if (!(p->radius >= 0.0f) || !(p->contact_offset >= 0.0f) || !(p->dt > 0.0f) || !(p->mass > 0.0f) || !(p->friction >= 0.0f) ||
        !(p->max_depenetration_velocity >= 0.0f) || p->iterations < 0)
        return agx_set_error(AGX_E_INVALID, "contact params out of range");
    if (num_envs == 0) return AGX_OK;
    if (!root_state || !contact_force || !crashes) return agx_set_error(AGX_E_NULL, "root_state/contact_force/crashes is NULL");
    if (root_state_stride < 13) return agx_set_error(AGX_E_INVALID, "root_state_stride < 13");
    *launch = true;
    return AGX_OK;
}

}  // namespace

extern "C" {

uint64_t agx_hp2_scene_bytes(int num_objects, int tris_per_object, int which) {
    int P = next_pow2(num_objects < 1 ? 1 : num_objects);
    switch (which) {
        case 0: return (uint64_t)num_objects * tris_per_object * kTriFloats * 4;
        case 1: return (uint64_t)(2 * P - 1) * kNodeFloats * 4;
        case 2: return (uint64_t)(P < 4 ? 4 : P) * 4;
        case 3: return (uint64_t)((num_objects + 3) / 4 * 4) * 4;
        case 4: return (uint64_t)num_objects * kObbFloats * 4;
        default: return 0;
    }
}

int agx_hp2_update_scene(const AgxHp2Scene* sc, const uint8_t* mask, void* stream) {
    int rc = validate_scene(sc);
    if (rc) return rc;
    if (sc->num_envs == 0) return AGX_OK;
    if (!sc->tmpl_tri_offset || !sc->tmpl_tris || !sc->tmpl_seg_base || !sc->tmpl_seg_mask || !sc->obj_pose || !sc->obj_template ||
        !sc->obj_seg_counter)
        return agx_set_error(AGX_E_NULL, "scene templates / instances are NULL");
    if (sc->obj_pose_stride < 7) return agx_set_error(AGX_E_INVALID, "obj_pose_stride < 7");
    const int K = sc->num_objects, P = sc->leaves_pow2;
    size_t smem = (size_t)(2 * P) * kNodeFloats * 4 + (size_t)P * 8 + (size_t)K * 6 * 4;
    rc = agx_check_cuda(cudaFuncSetAttribute(hp2_update_scene_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),
                        "cudaFuncSetAttribute(update_scene)");
    if (rc) return rc;
    hp2_update_scene_kernel<<<sc->num_envs, 256, smem, (cudaStream_t)stream>>>(*sc, mask);
    return agx_check_launch("hp2_update_scene_kernel");
}

int agx_hp2_collide(const AgxHp2Scene* sc, const float* robot_pose, int robot_pose_stride, float radius, uint8_t* crashes,
                    float* min_dist, void* stream) {
    int rc = validate_scene(sc);
    if (rc) return rc;
    if (sc->num_envs == 0) return AGX_OK;
    if (!robot_pose || !crashes) return agx_set_error(AGX_E_NULL, "robot_pose/crashes is NULL");
    if (robot_pose_stride < 3) return agx_set_error(AGX_E_INVALID, "robot_pose_stride < 3");
    if (!(radius >= 0.0f)) return agx_set_error(AGX_E_INVALID, "radius must be >= 0");
    hp2_collide_kernel<<<(sc->num_envs + 127) / 128, 128, 0, (cudaStream_t)stream>>>(*sc, robot_pose, robot_pose_stride, radius, crashes,
                                                                                  min_dist);
    return agx_check_launch("hp2_collide_kernel");
}

int agx_hp2_contact(const AgxHp2Scene* sc, int num_envs, const AgxContactParams* p, float* root_state, int root_state_stride,
                    float* contact_force, uint8_t* crashes, int32_t* contact_obj, void* stream) {
    AgxHp2Scene none = {};
    bool launch;
    int rc = contact_check(sc, num_envs, p, root_state, root_state_stride, contact_force, crashes, &launch);
    if (rc || !launch) return rc;
    hp2_contact_kernel<<<(num_envs + 127) / 128, 128, 0, (cudaStream_t)stream>>>(sc ? *sc : none, *p, num_envs, root_state,
                                                                                  root_state_stride, contact_force, crashes, contact_obj);
    return agx_check_launch("hp2_contact_kernel");
}

int agx_hp2_contact_moving(const AgxHp2Scene* sc, int num_envs, const AgxContactParams* p, const AgxContactMotion* m, float* root_state,
                           int root_state_stride, float* contact_force, uint8_t* crashes, int32_t* contact_obj, void* stream) {
    if (!sc) return agx_set_error(AGX_E_NULL, "scene is NULL: moving obstacles need a scene");
    if (!m) return agx_set_error(AGX_E_NULL, "motion is NULL");
    if (!m->asset_state || !m->obj_asset) return agx_set_error(AGX_E_NULL, "motion asset_state/obj_asset is NULL");
    if (m->asset_stride < 13) return agx_set_error(AGX_E_INVALID, "motion asset_stride < 13");
    if (m->num_assets < 1) return agx_set_error(AGX_E_INVALID, "motion num_assets < 1");
    bool launch;
    int rc = contact_check(sc, num_envs, p, root_state, root_state_stride, contact_force, crashes, &launch);
    if (rc || !launch) return rc;
    hp2_contact_moving_kernel<<<(num_envs + 127) / 128, 128, 0, (cudaStream_t)stream>>>(*sc, *p, *m, num_envs, root_state,
                                                                                         root_state_stride, contact_force, crashes,
                                                                                         contact_obj);
    return agx_check_launch("hp2_contact_moving_kernel");
}

int agx_hp2_contact_dynamic(const AgxHp2Scene* sc, int num_envs, const AgxContactParams* p, const AgxContactMotion* m,
                            const AgxObstacleMass* mass, float* root_state, int root_state_stride, float* contact_force, uint8_t* crashes,
                            int32_t* contact_obj, void* stream) {
    if (!sc) return agx_set_error(AGX_E_NULL, "scene is NULL: dynamic obstacles need a scene");
    if (!m) return agx_set_error(AGX_E_NULL, "motion is NULL");
    if (!m->asset_state || !m->obj_asset) return agx_set_error(AGX_E_NULL, "motion asset_state/obj_asset is NULL");
    if (m->asset_stride < 13) return agx_set_error(AGX_E_INVALID, "motion asset_stride < 13");
    if (m->num_assets < 1) return agx_set_error(AGX_E_INVALID, "motion num_assets < 1");
    if (!mass) return agx_set_error(AGX_E_NULL, "mass is NULL");
    bool launch;
    int rc = contact_check(sc, num_envs, p, root_state, root_state_stride, contact_force, crashes, &launch);
    if (rc || !launch) return rc;
    // the rows are written back: the caller's contract (aerial_gym_b200.h) is a writable asset_state buffer
    float* asset_state = const_cast<float*>(m->asset_state);
    hp2_contact_dynamic_kernel<<<(num_envs + 127) / 128, 128, 0, (cudaStream_t)stream>>>(*sc, *p, *m, asset_state, mass, num_envs,
                                                                                          root_state, root_state_stride, contact_force,
                                                                                          crashes, contact_obj);
    return agx_check_launch("hp2_contact_dynamic_kernel");
}

int agx_hp2_cast(const AgxHp2Scene* sc, const AgxHp2Sensor* sn, void* stream) {
    int rc = validate_scene(sc);
    if (rc) return rc;
    if (!sn) return agx_set_error(AGX_E_NULL, "sensor is NULL");
    if (sn->kind < AGX_SENSOR_CAMERA || sn->kind > AGX_SENSOR_NORMAL_FACEID_LIDAR) return agx_set_error(AGX_E_INVALID, "unknown sensor kind %d", sn->kind);
    if (sn->width < 1 || sn->height < 1 || sn->num_sensors < 1) return agx_set_error(AGX_E_INVALID, "sensor dims must be positive");
    if (sc->num_envs == 0) return AGX_OK;
    if (!sn->robot_pose || !sn->mount || !sn->pixels) return agx_set_error(AGX_E_NULL, "robot_pose/mount/pixels is NULL");
    if ((sn->kind == AGX_SENSOR_LIDAR || sn->kind == AGX_SENSOR_NORMAL_FACEID_LIDAR) && !sn->ray_table)
        return agx_set_error(AGX_E_NULL, "LiDAR needs ray_table");
    if (sn->robot_pose_stride < 7) return agx_set_error(AGX_E_INVALID, "robot_pose_stride < 7");
    int dev = 0, sms = 132, max_smem = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    const int W = sn->width, H = sn->height;
    // a work item = up to ~4096 rays of one (env, sensor) image (a 64x48 image is ONE item, so the
    // env's scene is staged once per image)
    int rows_per_item = 4096 / W;
    if (rows_per_item < 1) rows_per_item = 1;
    if (rows_per_item > H) rows_per_item = H;
    int items_per_image = (H + rows_per_item - 1) / rows_per_item;
    long long n_items = (long long)sc->num_envs * sn->num_sensors * items_per_image;
    size_t smem = scene_smem_bytes(sc->num_objects, sc->leaves_pow2, sc->tris_per_object, sc->obb != nullptr);
    bool use_smem = smem + 1024 <= (size_t)max_smem;
    cudaStream_t st = (cudaStream_t)stream;
    if (sc->num_meshes) {  // mesh objects: per-ray walk of the top level (staged when it fits) and of each reached BLAS (L2)
        auto kern = use_smem ? hp2_cast_kernel<true, false, true> : hp2_cast_kernel<false, false, true>;
        if (!use_smem) smem = 0;
        rc = agx_check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "cudaFuncSetAttribute(cast)");
        if (rc) return rc;
        int per_sm = 1;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kCastThreads, smem);
        if (per_sm < 1) per_sm = 1;
        long long grid = (long long)sms * per_sm;
        if (grid > n_items) grid = n_items;
        kern<<<(int)grid, kCastThreads, smem, st>>>(*sc, *sn, rows_per_item, items_per_image, n_items, 0);
        return agx_check_launch("hp2_cast_kernel");
    }
    const bool use_tile = use_smem && sc->leaves_pow2 <= kTileMaxLeaves &&
                          smem + record_smem_bytes(sc->num_objects) + 1024 <= (size_t)max_smem;
    if (use_tile) {  // small staged scenes: warp-per-tile candidate culling, no per-ray BVH walk
        smem += record_smem_bytes(sc->num_objects);
        rc = agx_check_cuda(cudaFuncSetAttribute(hp2_cast_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),
                            "cudaFuncSetAttribute(cast)");
        if (rc) return rc;
        int per_sm = 1;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, hp2_cast_kernel<true, true>, kCastThreads, smem);
        if (per_sm < 1) per_sm = 1;
        long long grid = (long long)sms * per_sm;
        if (grid > n_items) grid = n_items;
        hp2_cast_kernel<true, true><<<(int)grid, kCastThreads, smem, st>>>(*sc, *sn, rows_per_item, items_per_image, n_items, sc->num_objects);
    } else if (use_smem) {
        rc = agx_check_cuda(cudaFuncSetAttribute(hp2_cast_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),
                            "cudaFuncSetAttribute(cast)");
        if (rc) return rc;
        int per_sm = 1;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, hp2_cast_kernel<true>, kCastThreads, smem);
        if (per_sm < 1) per_sm = 1;
        long long grid = (long long)sms * per_sm;
        if (grid > n_items) grid = n_items;
        hp2_cast_kernel<true><<<(int)grid, kCastThreads, smem, st>>>(*sc, *sn, rows_per_item, items_per_image, n_items, 0);
    } else if (sn->kind == AGX_SENSOR_CAMERA || sn->kind == AGX_SENSOR_STEREO_CAMERA || sn->kind == AGX_SENSOR_NORMAL_FACEID_CAMERA) {
        // scene too large for shared memory, pinhole sensor: tile path with records only (see the kernel)
        const int cap = sc->num_objects < kBigSceneRecords ? sc->num_objects : kBigSceneRecords;
        smem = record_smem_bytes(cap);
        rc = agx_check_cuda(cudaFuncSetAttribute(hp2_cast_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),
                            "cudaFuncSetAttribute(cast)");
        if (rc) return rc;
        int per_sm = 1;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, hp2_cast_kernel<false, true>, kCastThreads, smem);
        if (per_sm < 1) per_sm = 1;
        long long grid = (long long)sms * per_sm;
        if (grid > n_items) grid = n_items;
        hp2_cast_kernel<false, true><<<(int)grid, kCastThreads, smem, st>>>(*sc, *sn, rows_per_item, items_per_image, n_items, cap);
    } else {
        int per_sm = 1;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, hp2_cast_kernel<false>, kCastThreads, 0);
        if (per_sm < 1) per_sm = 1;
        long long grid = (long long)sms * per_sm;
        if (grid > n_items) grid = n_items;
        hp2_cast_kernel<false><<<(int)grid, kCastThreads, 0, st>>>(*sc, *sn, rows_per_item, items_per_image, n_items, 0);
    }
    return agx_check_launch("hp2_cast_kernel");
}

}  // extern "C"
