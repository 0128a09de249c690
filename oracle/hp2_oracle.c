/*
 * HP2 oracle -- brute-force CPU restatement of the reference's ray-cast sensor path.
 *
 * TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline / --impl reference legs, never by the product.
 *
 * What it restates (reference = $AERIAL_GYM_REFERENCE/aerial_gym, commit f0d0f05):
 *   - sensor pose compose                  sensors/warp/warp_sensor.py:177-187
 *   - camera ray generation + outputs      sensors/warp/warp_kernels/warp_camera_kernels.py:13-66,125-282
 *   - LiDAR ray generation + outputs       sensors/warp/warp_kernels/warp_lidar_kernels.py:13-163
 *   - range limits / normalisation         sensors/warp/warp_sensor.py:202-225
 *   - vertex re-transform on reset         env_manager/warp_env_manager.py:40-54 (tf_apply, utils/math.py:313-320,374-376)
 *   - segmentation id of the hit face      warp_camera_kernels.py:277-279 (first vertex of the face)
 *
 * PARITY UNPINNED for the closest-hit query itself: the reference calls wp.mesh_query_ray
 * (warp-lang==1.0.0, requirements.txt:1), which is not in the tree and not installable here, and
 * the reference has no test or golden image for it.  The query is restated as the textbook
 * exhaustive Moller-Trumbore closest hit (two-sided, 0 <= t < max_t, ties -> lowest triangle
 * index).  Everything around the query follows the cited reference lines.
 *
 * Arithmetic contract with the CUDA kernel (csrc/hp2_raycast.cu): every multiply-add that may be
 * fused is written as an explicit fmaf() and this file is compiled with -ffp-contract=off (the
 * .cu with -fmad=false), division and sqrt are IEEE in both => depth and segmentation outputs
 * are BIT-IDENTICAL, independent of BVH traversal order.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define NO_HIT_RAY_VAL 1000.0f /* warp_camera_kernels.py:3 */
#define NO_HIT_SEG_VAL (-2)    /* warp_camera_kernels.py:4 */

typedef struct { float x, y, z; } v3;
typedef struct { float x, y, z, w; } q4;

static inline float dot3(v3 a, v3 b) { return fmaf(a.z, b.z, fmaf(a.y, b.y, a.x * b.x)); }
static inline v3 cross3(v3 a, v3 b) {
    v3 r;
    r.x = fmaf(a.y, b.z, -(a.z * b.y));
    r.y = fmaf(a.z, b.x, -(a.x * b.z));
    r.z = fmaf(a.x, b.y, -(a.y * b.x));
    return r;
}
static inline v3 sub3(v3 a, v3 b) { v3 r = {a.x - b.x, a.y - b.y, a.z - b.z}; return r; }
static inline v3 normalize3(v3 a) {
    float n = sqrtf(dot3(a, a));
    v3 r = {a.x / n, a.y / n, a.z / n};
    return r;
}
/* warp quat_rotate == utils/math.py:58-65:  v (2w^2-1) + 2w (q x v) + 2 q (q.v) */
static inline v3 quat_rotate(q4 q, v3 v) {
    v3 qv = {q.x, q.y, q.z};
    float s = fmaf(2.0f * q.w, q.w, -1.0f);
    v3 c = cross3(qv, v);
    float d2 = 2.0f * dot3(qv, v);
    float w2 = 2.0f * q.w;
    v3 r;
    r.x = fmaf(qv.x, d2, fmaf(c.x, w2, v.x * s));
    r.y = fmaf(qv.y, d2, fmaf(c.y, w2, v.y * s));
    r.z = fmaf(qv.z, d2, fmaf(c.z, w2, v.z * s));
    return r;
}
/* utils/math.py:313-320 quat_apply: v + w t + q x t, t = 2 (q x v) */
static inline v3 quat_apply(q4 q, v3 v) {
    v3 qv = {q.x, q.y, q.z};
    v3 c = cross3(qv, v);
    v3 t = {2.0f * c.x, 2.0f * c.y, 2.0f * c.z};
    v3 c2 = cross3(qv, t);
    v3 r;
    r.x = fmaf(q.w, t.x, v.x) + c2.x;
    r.y = fmaf(q.w, t.y, v.y) + c2.y;
    r.z = fmaf(q.w, t.z, v.z) + c2.z;
    return r;
}
/* utils/math.py:242-263 quat_mul */
static inline q4 quat_mul(q4 a, q4 b) {
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

/* ------------------------------------------------------------------------------------------
 * scene: world-space triangles per env (warp_env_manager.py:40-54)
 * tris layout: [n_envs][max_tris][9] = v0.xyz, e1.xyz, e2.xyz ; seg [n_envs][max_tris]
 * ------------------------------------------------------------------------------------------ */
void hp2o_build_world_tris(int n_envs, int n_obj, const float* obj_pose /*[E,K,7]*/,
                           const int32_t* obj_template /*[E,K]*/, const int32_t* obj_seg_counter /*[E,K]*/,
                           const int32_t* tmpl_tri_offset /*[T+1]*/, const float* tmpl_tris /*[Ft,9] v0,v1,v2*/,
                           const int32_t* tmpl_seg_base /*[Ft]*/, const int32_t* tmpl_seg_mask /*[Ft]*/,
                           int max_tris, float* out_tris, int32_t* out_seg, int32_t* out_count) {
    for (int e = 0; e < n_envs; ++e) {
        int n = 0;
        float* T = out_tris + (size_t)e * max_tris * 9;
        int32_t* S = out_seg + (size_t)e * max_tris;
        for (int k = 0; k < n_obj; ++k) {
            const float* p = obj_pose + ((size_t)e * n_obj + k) * 7;
            v3 t = {p[0], p[1], p[2]};
            q4 q = {p[3], p[4], p[5], p[6]};
            int tm = obj_template[(size_t)e * n_obj + k];
            int ctr = obj_seg_counter[(size_t)e * n_obj + k];
            for (int f = tmpl_tri_offset[tm]; f < tmpl_tri_offset[tm + 1]; ++f) {
                const float* tv = tmpl_tris + (size_t)f * 9;
                v3 a = {tv[0], tv[1], tv[2]}, b = {tv[3], tv[4], tv[5]}, c = {tv[6], tv[7], tv[8]};
                v3 wa = quat_apply(q, a), wb = quat_apply(q, b), wc = quat_apply(q, c); /* tf_apply = quat_apply + t */
                wa.x += t.x; wa.y += t.y; wa.z += t.z;
                wb.x += t.x; wb.y += t.y; wb.z += t.z;
                wc.x += t.x; wc.y += t.y; wc.z += t.z;
                v3 e1 = sub3(wb, wa), e2 = sub3(wc, wa);
                float* o = T + (size_t)n * 9;
                o[0] = wa.x; o[1] = wa.y; o[2] = wa.z;
                o[3] = e1.x; o[4] = e1.y; o[5] = e1.z;
                o[6] = e2.x; o[7] = e2.y; o[8] = e2.z;
                S[n] = tmpl_seg_base[f] + ctr * tmpl_seg_mask[f];
                ++n;
            }
        }
        out_count[e] = n;
    }
}

/* exhaustive closest hit; returns triangle index or -1 */
static int closest_hit(const float* T, int n, v3 o, v3 d, float max_t, float* t_out, v3* n_out) {
    int best = -1;
    float best_t = max_t;
    for (int i = 0; i < n; ++i) {
        const float* p = T + (size_t)i * 9;
        v3 v0 = {p[0], p[1], p[2]}, e1 = {p[3], p[4], p[5]}, e2 = {p[6], p[7], p[8]};
        v3 pv = cross3(d, e2);
        float det = dot3(e1, pv);
        if (fabsf(det) < 1e-20f) continue;
        float inv = 1.0f / det;
        v3 tv = sub3(o, v0);
        float u = dot3(tv, pv) * inv;
        if (u < 0.0f || u > 1.0f) continue;
        v3 qv = cross3(tv, e1);
        float v = dot3(d, qv) * inv;
        if (v < 0.0f || u + v > 1.0f) continue;
        float t = dot3(e2, qv) * inv;
        if (t < 0.0f || !(t < max_t)) continue;
        if (t < best_t || (t == best_t && best < 0)) { /* ascending scan: ties keep the lowest index */
            best_t = t;
            best = i;
        }
    }
    if (best >= 0) {
        *t_out = best_t;
        if (n_out) {
            const float* p = T + (size_t)best * 9;
            v3 e1 = {p[3], p[4], p[5]}, e2 = {p[6], p[7], p[8]};
            *n_out = normalize3(cross3(e1, e2));
        }
    }
    return best;
}

typedef struct Hp2oSensor {
    int32_t kind;            /* 0 camera, 1 lidar, 2 stereo camera, 3 normal+faceID camera, 4 normal+faceID lidar */
    int32_t width, height, num_sensors;
    int32_t calculate_depth; /* camera: depth (1) or range (0) image */
    int32_t return_pointcloud, pointcloud_in_world_frame, segmentation;
    int32_t fuse_epilogue;   /* apply range limits + normalisation (warp_sensor.py:202-225) */
    int32_t normalize_range;
    int32_t c_x, c_y;        /* warp_cam.py:63-64 */
    float kinv[9];           /* upper-left 3x3 of K_inv, row-major (warp_cam.py:43-62) */
    float far_plane;         /* = max_range (warp_cam.py:21) */
    float max_range, min_range, far_out_of_range_value, near_out_of_range_value;
    float frame_quat[4];     /* quat_from_euler(euler_frame_rot_deg) (warp_sensor.py:100-105) */
    float baseline;          /* stereo: config/sensor_config/camera_config/stereo_camera_config.py:9 */
    int32_t normal_in_world_frame; /* normal+faceID sensors (base_normal_faceID_camera_config.py) */
} Hp2oSensor;

static inline v3 kinv_mul(const float* k, v3 c) {
    v3 r;
    r.x = fmaf(k[2], c.z, fmaf(k[1], c.y, k[0] * c.x));
    r.y = fmaf(k[5], c.z, fmaf(k[4], c.y, k[3] * c.x));
    r.z = fmaf(k[8], c.z, fmaf(k[7], c.y, k[6] * c.x));
    return r;
}
static inline float range_epilogue(const Hp2oSensor* s, float px) {
    /* warp_sensor.py:216-225: two sequential masked assignments, then the division */
    if (px > s->max_range) px = s->far_out_of_range_value;
    if (px < s->min_range) px = s->near_out_of_range_value;
    if (s->normalize_range && !s->pointcloud_in_world_frame) px = px / s->max_range;
    return px;
}

/* robot_pose [E,7] (pos, quat xyzw); mount [E,S,7] local pos + local quat; ray_table [H,W,3] (lidar)
 * pixels: [E,S,H,W] or [E,S,H,W,3]; seg: [E,S,H,W] or NULL */
void hp2o_cast(const Hp2oSensor* s, int n_envs, const float* robot_pose, const float* mount, const float* ray_table,
               const float* tris, const int32_t* seg_ids, const int32_t* tri_count, int max_tris, float* pixels,
               int32_t* seg) {
    const int W = s->width, H = s->height, S = s->num_sensors;
    q4 qf = {s->frame_quat[0], s->frame_quat[1], s->frame_quat[2], s->frame_quat[3]};
    /* threads: the Python wrapper splits envs across a thread pool (ctypes releases the GIL) */
    for (int e = 0; e < n_envs; ++e) {
        const float* rp = robot_pose + (size_t)e * 7;
        v3 rpos = {rp[0], rp[1], rp[2]};
        q4 rq = {rp[3], rp[4], rp[5], rp[6]};
        const float* T = tris + (size_t)e * max_tris * 9;
        const int32_t* SG = seg_ids + (size_t)e * max_tris;
        const int nt = tri_count[e];
        for (int c = 0; c < S; ++c) {
            const float* m = mount + ((size_t)e * S + c) * 7;
            v3 lp = {m[0], m[1], m[2]};
            q4 lq = {m[3], m[4], m[5], m[6]};
            /* warp_sensor.py:180-187 */
            v3 sp = quat_apply(rq, lp);
            sp.x += rpos.x; sp.y += rpos.y; sp.z += rpos.z;
            q4 sq = quat_mul(rq, quat_mul(lq, qf));
            v3 rd_p = {0, 0, 0};
            const int is_cam = (s->kind == 0 || s->kind == 2 || s->kind == 3);
            const int norm_uv = s->return_pointcloud || s->kind == 3; /* pointcloud + normal kernels normalise uv */
            v3 stereo_pos = sp;
            if (s->kind == 2) {
                v3 off = {-s->baseline, 0.0f, 0.0f};
                v3 ro = quat_rotate(sq, off);
                stereo_pos.x = sp.x + ro.x; stereo_pos.y = sp.y + ro.y; stereo_pos.z = sp.z + ro.z;
            }
            if (is_cam) {
                v3 cp = {(float)s->c_x, (float)s->c_y, 1.0f};
                v3 uvp = kinv_mul(s->kinv, cp);
                if (norm_uv) uvp = normalize3(uvp);
                rd_p = normalize3(quat_rotate(sq, uvp));
            }
            for (int y = 0; y < H; ++y) {
                for (int x = 0; x < W; ++x) {
                    v3 uv, rd;
                    float mult = 1.0f, max_t = s->far_plane;
                    if (is_cam) {
                        v3 cc = {(float)x, (float)y, 1.0f};
                        uv = kinv_mul(s->kinv, cc);
                        if (norm_uv) uv = normalize3(uv); /* quirk: only the pointcloud / normal kernels normalise uv */
                        rd = normalize3(quat_rotate(sq, uv));
                        if (s->kind != 3 && !s->return_pointcloud && s->calculate_depth) {
                            mult = dot3(rd, rd_p);
                            max_t = s->far_plane / mult; /* warp_camera_kernels.py:221,275 */
                        }
                    } else {
                        const float* rt = ray_table + ((size_t)y * W + x) * 3;
                        v3 r0 = {rt[0], rt[1], rt[2]};
                        uv = normalize3(r0); /* warp_lidar_kernels.py:31-33 */
                        rd = normalize3(quat_rotate(sq, uv));
                    }
                    float t = 0.0f;
                    v3 nrm = {0.0f, 0.0f, 0.0f};
                    int hit = closest_hit(T, nt, sp, rd, max_t, &t, &nrm);
                    float dist = NO_HIT_RAY_VAL;
                    int32_t sv = NO_HIT_SEG_VAL;
                    size_t pix = (((size_t)e * S + c) * H + y) * W + x;
                    if (s->kind == 3 || s->kind == 4) {
                        /* normal + face id: warp_camera_kernels.py:70-121, warp_lidar_kernels.py:90-126 */
                        v3 o = {0.0f, 0.0f, 0.0f};
                        if (hit >= 0) {
                            if (s->normal_in_world_frame) o = nrm;
                            else if (s->kind == 3) {
                                v3 ez = {0.0f, 0.0f, 1.0f}, ey = {0.0f, 1.0f, 0.0f};
                                o.x = dot3(nrm, rd_p); o.y = dot3(nrm, cross3(rd_p, ez)); o.z = dot3(nrm, cross3(rd_p, ey));
                            } else {
                                q4 qi = {-sq.x, -sq.y, -sq.z, sq.w};
                                o = normalize3(quat_rotate(qi, nrm));
                            }
                        }
                        pixels[pix * 3 + 0] = o.x; pixels[pix * 3 + 1] = o.y; pixels[pix * 3 + 2] = o.z;
                        if (seg) seg[pix] = hit;  /* face index, -1 on a miss */
                        continue;
                    }
                    if (s->kind == 2) {
                        /* stereo occlusion: warp_stereo_camera_kernels.py:205-222 */
                        float t2;
                        v3 ep, dv, rrev;
                        dist = -1.0f; /* INVALID_PIXEL_VAL */
                        if (hit >= 0) {
                            ep.x = fmaf(rd.x * t, 0.999f, sp.x); ep.y = fmaf(rd.y * t, 0.999f, sp.y); ep.z = fmaf(rd.z * t, 0.999f, sp.z);
                            dv = sub3(stereo_pos, ep);
                            float dl = sqrtf(dot3(dv, dv));
                            rrev = normalize3(dv);
                            if (closest_hit(T, nt, ep, rrev, dl, &t2, NULL) < 0) { dist = t * mult; sv = SG[hit]; }
                        } else {
                            ep.x = sp.x + (rd.x * s->far_plane) / mult; ep.y = sp.y + (rd.y * s->far_plane) / mult; ep.z = sp.z + (rd.z * s->far_plane) / mult;
                            dv = sub3(stereo_pos, ep);
                            float dl = sqrtf(dot3(dv, dv));
                            rrev = normalize3(dv);
                            if (closest_hit(T, nt, ep, rrev, dl, &t2, NULL) < 0) dist = NO_HIT_RAY_VAL;
                        }
                        pixels[pix] = s->fuse_epilogue ? range_epilogue(s, dist) : dist;
                        if (seg) seg[pix] = sv;
                        continue;
                    }
                    if (hit >= 0) {
                        dist = mult * t;
                        sv = SG[hit];
                    }
                    if (s->return_pointcloud) {
                        v3 p;
                        if (s->pointcloud_in_world_frame) {
                            p.x = fmaf(dist, rd.x, sp.x); p.y = fmaf(dist, rd.y, sp.y); p.z = fmaf(dist, rd.z, sp.z);
                        } else {
                            p.x = dist * uv.x; p.y = dist * uv.y; p.z = dist * uv.z;
                        }
                        if (s->fuse_epilogue && !s->pointcloud_in_world_frame) {
                            /* warp_sensor.py:203-215: norm-based clipping of the whole point */
                            float nrm2 = sqrtf(dot3(p, p));
                            if (nrm2 > s->max_range) { p.x = p.y = p.z = s->far_out_of_range_value; }
                            nrm2 = sqrtf(dot3(p, p));
                            if (nrm2 < s->min_range) { p.x = p.y = p.z = s->near_out_of_range_value; }
                            if (s->normalize_range) { p.x /= s->max_range; p.y /= s->max_range; p.z /= s->max_range; }
                        }
                        pixels[pix * 3 + 0] = p.x; pixels[pix * 3 + 1] = p.y; pixels[pix * 3 + 2] = p.z;
                    } else {
                        pixels[pix] = s->fuse_epilogue ? range_epilogue(s, dist) : dist;
                    }
                    if (seg) seg[pix] = sv;
                }
            }
        }
    }
}

/* ------------------------------------------------------------------------------------------
 * a14: collision flag.  Reference: EnvManager.compute_observations (env_manager/env_manager.py:358-362)
 * thresholds the PhysX contact force on body 0; PhysX is not in the tree, so the flag is restated
 * geometrically (DESIGN.md): the robot's base-link collision sphere overlaps the env's triangle
 * mesh  <=>  min over triangles of |closest_point(tri, c) - c|^2 <= r^2.  Closest point on a
 * triangle: Ericson, Real-Time Collision Detection 5.1.5 (Voronoi-region form).
 * Same explicit-fmaf arithmetic contract as the ray path => flags are bit-exact.
 * ------------------------------------------------------------------------------------------ */
static float point_tri_dist2(v3 p, v3 a, v3 ab, v3 ac) {
    v3 ap = sub3(p, a);
    float d1 = dot3(ab, ap), d2 = dot3(ac, ap);
    if (d1 <= 0.0f && d2 <= 0.0f) return dot3(ap, ap);
    v3 b = {a.x + ab.x, a.y + ab.y, a.z + ab.z};
    v3 bp = sub3(p, b);
    float d3 = dot3(ab, bp), d4 = dot3(ac, bp);
    if (d3 >= 0.0f && d4 <= d3) return dot3(bp, bp);
    float vc = fmaf(d1, d4, -(d3 * d2));
    if (vc <= 0.0f && d1 >= 0.0f && d3 <= 0.0f) {
        float v = d1 / (d1 - d3);
        v3 q = {fmaf(v, ab.x, a.x), fmaf(v, ab.y, a.y), fmaf(v, ab.z, a.z)};
        v3 d = sub3(p, q);
        return dot3(d, d);
    }
    v3 c = {a.x + ac.x, a.y + ac.y, a.z + ac.z};
    v3 cp = sub3(p, c);
    float d5 = dot3(ab, cp), d6 = dot3(ac, cp);
    if (d6 >= 0.0f && d5 <= d6) return dot3(cp, cp);
    float vb = fmaf(d5, d2, -(d1 * d6));
    if (vb <= 0.0f && d2 >= 0.0f && d6 <= 0.0f) {
        float w = d2 / (d2 - d6);
        v3 q = {fmaf(w, ac.x, a.x), fmaf(w, ac.y, a.y), fmaf(w, ac.z, a.z)};
        v3 d = sub3(p, q);
        return dot3(d, d);
    }
    float va = fmaf(d3, d6, -(d5 * d4));
    if (va <= 0.0f && (d4 - d3) >= 0.0f && (d5 - d6) >= 0.0f) {
        float w = (d4 - d3) / ((d4 - d3) + (d5 - d6));
        v3 bc = sub3(c, b);
        v3 q = {fmaf(w, bc.x, b.x), fmaf(w, bc.y, b.y), fmaf(w, bc.z, b.z)};
        v3 d = sub3(p, q);
        return dot3(d, d);
    }
    float denom = 1.0f / (va + vb + vc);
    float v = vb * denom, w = vc * denom;
    v3 q = {fmaf(w, ac.x, fmaf(v, ab.x, a.x)), fmaf(w, ac.y, fmaf(v, ab.y, a.y)), fmaf(w, ac.z, fmaf(v, ab.z, a.z))};
    v3 d = sub3(p, q);
    return dot3(d, d);
}

/* robot_pose [E,7]; flags [E] u8 (1 = overlap); min_dist2 [E] (FLT_MAX-like 3.0e38 when no triangle) */
void hp2o_collide(int n_envs, const float* robot_pose, float radius, const float* tris, const int32_t* tri_count,
                  int max_tris, uint8_t* flags, float* min_dist2) {
    float r2 = radius * radius;
    for (int e = 0; e < n_envs; ++e) {
        const float* rp = robot_pose + (size_t)e * 7;
        v3 c = {rp[0], rp[1], rp[2]};
        const float* T = tris + (size_t)e * max_tris * 9;
        float best = 3.0e38f;
        for (int i = 0; i < tri_count[e]; ++i) {
            const float* p = T + (size_t)i * 9;
            v3 a = {p[0], p[1], p[2]}, ab = {p[3], p[4], p[5]}, ac = {p[6], p[7], p[8]};
            float d2 = point_tri_dist2(c, a, ab, ac);
            if (d2 < best) best = d2;
        }
        flags[e] = best <= r2 ? 1 : 0;
        if (min_dist2) min_dist2[e] = best;
    }
}

int hp2o_sizeof_sensor(void) { return (int)sizeof(Hp2oSensor); }
