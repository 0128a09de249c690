// HP1: fused multirotor step for sm_90a (H100).
//
//   update_states -> Lee controller -> allocation -> motor model -> drag/disturbance ->
//   rigid-body integrate  (x physics_steps)  [-> position-task reward / flags / reset / obs]
//
// One thread per environment, one warp per 32-env tile.  The [N,13] AoS root-state rows the
// reference API exposes (IGE_env_manager.py:301-311, views must stay views) are moved with
// coalesced 16-byte loads of the contiguous 32x13 tile into shared memory and read back
// conflict-free (row stride 13 is coprime with the 32 banks); [N,4]/[N,8] arrays are one or
// two float4 per thread.  No tensor-core path: per-env work is <= 8x6 contractions.
//
// Reference functions restated here are cited inline (paths relative to aerial_gym/).
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#ifdef AGX_TIMELINE
#include <chrono>
#endif

#include "../../include/aerial_gym_b200.h"
#include "agx_common.cuh"
#include "agx_math.cuh"
#include "hp1_core.cuh"
#include "disturbance_core.cuh"

using namespace agx;

namespace {

#ifndef AGX_HP1_WARPS_PER_BLOCK
#define AGX_HP1_WARPS_PER_BLOCK 2
#endif
constexpr int kWarpsPerBlock = AGX_HP1_WARPS_PER_BLOCK;
constexpr int kThreads = kWarpsPerBlock * 32;
constexpr int kTileFloats = 32 * 13;


// The chain handshake polls with RELAXED loads and acquires once, with a fence, after the wait: on sm_90a every acquire (an
// ld.acquire, or the acquire half of fence.acq_rel) is followed by CCTL.IVALL, which invalidates the SM's whole L1 -- and with it the
// stack lines of every warp on the SM.  fence.acquire costs that invalidation once per wait instead of once per poll, and
// fence.release is a MEMBAR without one.
__device__ __forceinline__ void fence_acquire_gpu() { asm volatile("fence.acquire.gpu;" ::: "memory"); }
__device__ __forceinline__ void fence_release_gpu() { asm volatile("fence.release.gpu;" ::: "memory"); }
__device__ __forceinline__ void st_relaxed_gpu_u32(uint32_t* p, uint32_t v) {
    asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_relaxed_gpu_u32(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long ld_relaxed_gpu_u64(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void red_relaxed_gpu_add_u32(uint32_t* p, uint32_t v) {
    asm volatile("red.relaxed.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// Every in-kernel wait of the chained step is bounded by WALL-CLOCK time (%globaltimer), not by a poll count, and never traps:
// on expiry the warp records AGX_HP1_ERR_TIMEOUT in the engine's error word (any_reset[2]) and goes on, later waits give up at
// once, and the host reports AGX_E_TIMEOUT at its next agx_hp1_check() -- a slow neighbour kernel or a late peer costs a failed
// run, not a poisoned CUDA context.  agx_set_spin_timeout_ms() changes the bound (default 20 s).
__device__ unsigned long long g_hp1_spin_timeout_ns = 20ull * 1000ull * 1000ull * 1000ull;
constexpr int kErrWord = 2;  // index into any_reset[]
// error word = code | step << 4: 1 = the tile's previous step never published, 2 = step T-2 never completed, 3 = the reset decision
// never closed (not every warp of the step arrived: the grid was not fully resident)
template <class Pred>
__device__ __forceinline__ bool spin_until(Pred ok, int32_t* any_reset, int code) {
    if (ok()) return true;
    volatile int32_t* err = any_reset + kErrWord;
    if (*err) return false;
    const long long t0 = clock64();
    const long long limit = (long long)g_hp1_spin_timeout_ns * 2;  // ns -> SM cycles at <= 2 GHz; clock64 is monotonic per SM (%globaltimer may be re-synchronised and jump)
    unsigned polls = 0;
    while (!ok()) {
        if ((++polls & 255u) == 0u) {
            if (*err) return false;
            if (clock64() - t0 > limit) {
                atomicCAS(any_reset + kErrWord, 0, code);
                return false;
            }
        }
    }
    return true;
}

// ---- tile IO ---------------------------------------------------------------------------
// rows [env0, env0+n_valid) of a dense [N,13] array -> the tile (row `lane` for lane `lane`)
__device__ __forceinline__ void fill_rows13(const float* __restrict__ base, int env0, int n_valid, float* tile, int lane,
                                            bool vec_ok) {
    const float* src = base + (size_t)env0 * 13;
    if (n_valid == 32 && vec_ok) {
        const float4* s4 = reinterpret_cast<const float4*>(src);
        float4* t4 = reinterpret_cast<float4*>(tile);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            int idx = lane + 32 * i;
            if (idx < kTileFloats / 4) t4[idx] = __ldcg(s4 + idx);  // L2 (see "chained steps": never a stale L1 line)
        }
    } else {
        int n = n_valid * 13;
        for (int i = lane; i < n; i += 32) tile[i] = __ldcg(src + i);
    }
    __syncwarp();
}
// rows [env0, env0+n_valid) of a dense [N,13] array -> this lane's row in r[13]
__device__ __forceinline__ void load_rows13(const float* __restrict__ base, int env0, int n_valid,
                                            float* tile, int lane, float r[13], bool vec_ok) {
    fill_rows13(base, env0, n_valid, tile, lane, vec_ok);
    if (lane < n_valid) {
#pragma unroll
        for (int j = 0; j < 13; ++j) r[j] = tile[lane * 13 + j];
    }
    __syncwarp();
}
// the tile (row `lane` written by lane `lane`) -> rows [env0, env0+n_valid) of a dense [N,13] array
__device__ __forceinline__ void flush_rows13(float* __restrict__ base, int env0, int n_valid, const float* tile, int lane,
                                             bool vec_ok) {
    __syncwarp();
    float* dst = base + (size_t)env0 * 13;
    if (n_valid == 32 && vec_ok) {
        float4* d4 = reinterpret_cast<float4*>(dst);
        const float4* t4 = reinterpret_cast<const float4*>(tile);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            int idx = lane + 32 * i;
            if (idx < kTileFloats / 4) d4[idx] = t4[idx];
        }
    } else {
        int n = n_valid * 13;
        for (int i = lane; i < n; i += 32) dst[i] = tile[i];
    }
    __syncwarp();
}
__device__ __forceinline__ void store_rows13(float* __restrict__ base, int env0, int n_valid, float* tile,
                                             int lane, const float r[13], bool vec_ok) {
    if (lane < n_valid) {
#pragma unroll
        for (int j = 0; j < 13; ++j) tile[lane * 13 + j] = r[j];
    }
    flush_rows13(base, env0, n_valid, tile, lane, vec_ok);
}
template <int M>
__device__ __forceinline__ void load_m(const float* __restrict__ p, int env, float out[M]) {
    if constexpr (M % 4 == 0) {
        const float4* p4 = reinterpret_cast<const float4*>(p + (size_t)env * M);
#pragma unroll
        for (int i = 0; i < M / 4; ++i) {
            float4 v = __ldcg(p4 + i);
            out[4 * i] = v.x; out[4 * i + 1] = v.y; out[4 * i + 2] = v.z; out[4 * i + 3] = v.w;
        }
    } else {
#pragma unroll
        for (int i = 0; i < M; ++i) out[i] = __ldcg(p + (size_t)env * M + i);
    }
}
template <int M>
__device__ __forceinline__ void store_m(float* __restrict__ p, int env, const float in[M]) {
    if constexpr (M % 4 == 0) {
        float4* p4 = reinterpret_cast<float4*>(p + (size_t)env * M);
#pragma unroll
        for (int i = 0; i < M / 4; ++i) p4[i] = make_float4(in[4 * i], in[4 * i + 1], in[4 * i + 2], in[4 * i + 3]);
    } else {
#pragma unroll
        for (int i = 0; i < M; ++i) p[(size_t)env * M + i] = in[i];
    }
}
__device__ __forceinline__ void st3(float* p, int env, V3 v) {
    p[(size_t)env * 3 + 0] = v.x; p[(size_t)env * 3 + 1] = v.y; p[(size_t)env * 3 + 2] = v.z;
}



template <int M>
__device__ __forceinline__ void load_params(const AgxHp1Config& cfg, const AgxHp1Buffers& buf, int env, EnvParams<M>& p) {
    load_m<M>(buf.motor_thrust, env, p.thrust);
    if (buf.tau_inc) load_m<M>(buf.tau_inc, env, p.tau_inc);
    else {
#pragma unroll
        for (int i = 0; i < M; ++i) p.tau_inc[i] = cfg.tau_inc;
    }
    if (buf.tau_dec) load_m<M>(buf.tau_dec, env, p.tau_dec);
    else {
#pragma unroll
        for (int i = 0; i < M; ++i) p.tau_dec[i] = cfg.tau_dec;
    }
    if (buf.k_thrust) load_m<M>(buf.k_thrust, env, p.k);
    else {
#pragma unroll
        for (int i = 0; i < M; ++i) p.k[i] = cfg.k_thrust;
    }
    p.g.kp = buf.K_pos ? ld3cg(buf.K_pos + (size_t)env * 3) : ld3c(cfg.K_pos);
    p.g.kv = buf.K_vel ? ld3cg(buf.K_vel + (size_t)env * 3) : ld3c(cfg.K_vel);
    p.g.kr = buf.K_rot ? ld3cg(buf.K_rot + (size_t)env * 3) : ld3c(cfg.K_rot);
    p.g.kw = buf.K_angvel ? ld3cg(buf.K_angvel + (size_t)env * 3) : ld3c(cfg.K_angvel);
}
template <int M>
__device__ __forceinline__ void store_reset_params(const AgxHp1Buffers& buf, int env, const EnvParams<M>& p) {
    if (buf.tau_inc) store_m<M>(buf.tau_inc, env, p.tau_inc);
    if (buf.tau_dec) store_m<M>(buf.tau_dec, env, p.tau_dec);
    if (buf.k_thrust) store_m<M>(buf.k_thrust, env, p.k);
    if (buf.K_pos) st3(buf.K_pos, env, p.g.kp);
    if (buf.K_vel) st3(buf.K_vel, env, p.g.kv);
    if (buf.K_rot) st3(buf.K_rot, env, p.g.kr);
    if (buf.K_angvel) st3(buf.K_angvel, env, p.g.kw);
    if (buf.bounds_min) st3(buf.bounds_min, env, p.bmin);
    if (buf.bounds_max) st3(buf.bounds_max, env, p.bmax);
}
__device__ __forceinline__ void store_derived(const AgxHp1Buffers& buf, int env, const Derived& d) {
    if (buf.euler) st3(buf.euler, env, d.euler);
    if (buf.vehicle_orientation)
        reinterpret_cast<float4*>(buf.vehicle_orientation)[env] = make_float4(d.qveh.x, d.qveh.y, d.qveh.z, d.qveh.w);
    if (buf.vehicle_linvel) st3(buf.vehicle_linvel, env, d.vveh);
    if (buf.body_linvel) st3(buf.body_linvel, env, d.vb);
    if (buf.body_angvel) st3(buf.body_angvel, env, d.wb);
}

// in-kernel reset of env `env0 + owner` (a15), warp-cooperative: every lane evaluates one Philox block, the owner applies them.
// Rare (an env resets every ~500 steps) and ~800 instructions: -DAGX_HP1_NOINLINE_RESET keeps it out of the step's straight line.
#ifdef AGX_HP1_NOINLINE_RESET
#define AGX_HP1_RESET_FN __device__ __noinline__
#else
#define AGX_HP1_RESET_FN __device__ __forceinline__
#endif
template <int M>
AGX_HP1_RESET_FN void reset_one_env(const AgxHp1Config& cfg, const AgxHp1Buffers& buf, int env0, int owner, uint32_t ep, int lane, float* tile,
                                    EnvState& s, EnvParams<M>& p) {
    coop_rng_draw<M>(cfg, (uint32_t)(cfg.env_id_offset + env0 + owner), ep, lane, tile);
    __syncwarp();
    if (lane == owner) {
        const int env = env0 + owner;
        apply_reset_from_tile<M>(cfg, tile, s, p);
        buf.episode_count[env] = ep + 1u;
        store_reset_params<M>(buf, env, p);
    }
    __syncwarp();
}

// =========================================================================================
// main kernel
// =========================================================================================
// 8 CTAs/SM -> <= 128 registers: all 1024 CTAs of the 65,536-env launch are resident in one wave
// COOP (grid <= one resident wave, so all CTAs are co-resident; one tile per warp).
//
// (1) The stale-observation quirk ("a reset anywhere refreshes everybody", base_multirotor.py:204-205) is
// resolved inside the kernel with a one-sided grid barrier instead of a second launch:
//   * a warp that sees at its START that one of its envs truncates this step (sim_steps + 1 > episode
//     length) raises the step's flag right away; crashes raise it in the epilogue;
//   * every warp reads the flag when its physics is done (the load overlaps the epilogue).  Flag up
//     (monotonic) -> everybody is refreshed: no waiting, no synchronisation at all.  With staggered
//     episodes some env truncates every step, so this is the steady state;
//   * flag still down: the warp counts itself in and waits until the flag rises OR all warps of the step
//     have arrived (= nobody reset);
//   * the observation (and the derived arrays) are written once, after the decision.
//
// (2) Chained steps.  Env i's step T+1 depends on env i's step T only, so consecutive step launches are
// chained per TILE, not per grid: launched with programmatic stream serialization, a step's CTAs are
// scheduled while the previous step's slower warps are still running, each warp takes its step number T
// from the launch (the host counts chained launches: Hp1Engine._chain_T) and counts its claim on a per-tile claim counter with a
// non-returning reduction -- or, for a caller that does not count (step == kClaimOnDevice), takes T from the claim counter (atomicAdd,
// before the CTA triggers its dependents, so claims are in launch order) --, spins until its tile's done-counter says step T-1 has been published (fence.release after the last
// store / relaxed polls, then one fence.acquire before the first L2-only load), and runs.  The launch's tail (slow SMs, the ~6 % of
// warps with a resetting env) no longer gates the next step.  A warp also waits until step T-2 is complete
// everywhere, so at most two consecutive steps are in flight and four parity slots suffice:
//   any_reset[4 + (T & 3)]        u32 flag of step T: raised = holds T + 1 (monotonic, never cleared)
//   any_reset[8 + 2 * (T & 3)]    u64 arrivals of the steps = T mod 4 (cumulative, never cleared): "this warp's physics and reset
//                                 decision are done" -- in the rare no-reset-yet case counted BEFORE the observation is written
//   publish_ctr[T & 3]            u64 published tiles of the steps = T mod 4 (cumulative; optional, on a cache line of its own --
//                                 the arrival line is hammered by 2048 atomics and their pollers per step, a second atomic per warp
//                                 on it cost the dependent-chain loop 2.5 us): "this tile's state, observation, reward and flags
//                                 are in memory" -- what a consumer outside the kernel (agx_obs_gather_push) waits on
//   tile_sync[tile], tile_sync[n_tiles + tile]   claim / done counters of the tile
// (3) Multi-GPU: the step kernel never touches NVLink and never waits for the gather.  With an observation all-gather attached
// (agx_obs_gather_push, p2p_allgather.cu, on side streams) buf.obs is one slot of a ring the push kernels read asynchronously; the
// HOST keeps a step from overwriting a slot whose push has not finished (stream events) -- an in-kernel wait here would let the
// blocked step's CTAs and their chained successors hold every CTA slot the pending push needs (a deadlock until the wall-clock
// bound fires: tests/test_gather_protocol_model.py).
#ifdef AGX_TIMELINE  // debug builds only (tools/dbg/timeline.py, tools/step_breakdown.py): per-warp globaltimer stamps
// 0 start, 1 physics done, 2 epilogue done, 3 end; chained steps: 4 step index known (claim), 5 waits done, 6 first loads arrived
__device__ unsigned long long g_timeline[7][8192];
__device__ __forceinline__ unsigned long long gtimer() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
#define AGX_TL(slot) do { if (lane == 0) { int w_ = blockIdx.x * kWarpsPerBlock + warp; if (w_ < 8192) g_timeline[slot][w_] = gtimer(); } } while (0)
#else
#define AGX_TL(slot) do { } while (0)
#endif

#ifndef AGX_HP1_MIN_BLOCKS
#define AGX_HP1_MIN_BLOCKS (16 / AGX_HP1_WARPS_PER_BLOCK)  // 16 warps x 128 registers = the register file
#endif
constexpr uint32_t kClaimOnDevice = 0xffffffffu;  // `step` of a chained launch whose caller does not count its launches
template <int M, bool TASK, bool COOP = false, int SPEC = -1>
__global__ void __launch_bounds__(kThreads, AGX_HP1_MIN_BLOCKS)
hp1_step_kernel(const __grid_constant__ AgxHp1Config cfg, const __grid_constant__ AgxHp1Buffers buf, int vec_ok, uint32_t step) {
    using SP = HpSpec<SPEC>;
    __shared__ __align__(16) float tiles[kWarpsPerBlock][kTileFloats];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float* tile = tiles[warp];
    const int N = cfg.num_envs;
    const int n_tiles = (N + 31) >> 5;
    const int A = cfg.num_actions;
    AGX_TL(0);
    uint32_t* reset_flag = reinterpret_cast<uint32_t*>(buf.any_reset);
    unsigned long long* arrive_ctr = nullptr;
    unsigned long long arrive_target = 0;  // arrivals once every warp of this step has counted itself in
    uint32_t step_T = 0;
    if constexpr (COOP) {
        const int my_tile = blockIdx.x * kWarpsPerBlock + warp;
        const bool has_tile = my_tile < n_tiles;
        if (step != kClaimOnDevice) {
            // the host knows T: no round trip before the waits, and the next step's CTAs may be scheduled at once (programmatic
            // dependent launch: once every CTA of this grid is here).  The claim is still counted, so tile_sync reads the same.
            asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
            step_T = step;
            if (has_tile && lane == 0) red_relaxed_gpu_add_u32(buf.tile_sync + my_tile, 1u);
        } else {
            if (has_tile && lane == 0) step_T = atomicAdd(buf.tile_sync + my_tile, 1u);  // claim: which step of this tile am I?
            step_T = __shfl_sync(0xffffffffu, step_T, 0);
            __syncthreads();  // every warp of the CTA holds its claim before the CTA lets the next launch in
            asm volatile("griddepcontrol.launch_dependents;" ::"r"(step_T) : "memory");
        }
        AGX_TL(4);
        if (has_tile) {
            if (lane == 0) {
                // the tile's previous step has published its state, and step T-2 is complete everywhere (bounds the skew to two steps
                // in flight).  Both counters are loaded at once, so the common case -- both already satisfied -- costs one round trip.
                // Only the one arrival counter T selects is read: extra loads on the line the arrival atomics hammer slow the
                // dependent-chain loop.
                const uint32_t* done = buf.tile_sync + n_tiles + my_tile;
                const uint32_t P = step_T - 2u;
                const unsigned long long* a2 = reinterpret_cast<const unsigned long long*>(buf.any_reset + 8) + (P & 3u);
                const unsigned long long want2 = step_T >= 2u ? (unsigned long long)(P / 4u + 1u) * (unsigned long long)n_tiles : 0ull;
                const uint32_t done0 = ld_relaxed_gpu_u32(done);
                const unsigned long long arrived0 = step_T >= 2u ? ld_relaxed_gpu_u64(a2) : 0ull;
                if (done0 != step_T)
                    spin_until([&] { return ld_relaxed_gpu_u32(done) == step_T; }, buf.any_reset, 1 | (int)(step_T << 4));
                if (arrived0 < want2)
                    spin_until([&] { return ld_relaxed_gpu_u64(a2) >= want2; }, buf.any_reset, 2 | (int)(step_T << 4));
                fence_acquire_gpu();  // one acquire for both waits, before the warp's first load of the tile
            }
            __syncwarp();
        }
        AGX_TL(5);
        reset_flag = reinterpret_cast<uint32_t*>(buf.any_reset) + 4 + (step_T & 3u);
        arrive_ctr = reinterpret_cast<unsigned long long*>(buf.any_reset + 8) + (step_T & 3u);
        arrive_target = (unsigned long long)(step_T / 4u + 1u) * (unsigned long long)n_tiles;
    }
    const uint32_t flag_tag = step_T + 1u;
    bool warp_raised = false;
    EnvState s;
    Derived d;
    V3 tgt{0.f, 0.f, 0.f};
    float o[13];

    for (int t = blockIdx.x * kWarpsPerBlock + warp; t < n_tiles; t += gridDim.x * kWarpsPerBlock) {
        const int env0 = t << 5;
        const int n_valid = min(32, N - env0);
        const int env = env0 + lane;
        const bool valid = lane < n_valid;

        // every global load of the step is issued here, before the first use, so their DRAM
        // latencies overlap (the kernel is latency bound at 65,536 envs)
        EnvParams<M> p;
        float act[AGX_MAX_MOTORS];
        int steps_in = 0;
        tgt = V3{0.f, 0.f, 0.f};
        if (valid) {
            load_params<M>(cfg, buf, env, p);
            if constexpr (TASK) {
                steps_in = __ldcg(buf.sim_steps + env);
                if (buf.target_position) tgt = ld3cg(buf.target_position + (size_t)env * 3);
            }
            if (A == 4) {
                float4 a4 = __ldcg(reinterpret_cast<const float4*>(buf.actions) + env);
                act[0] = a4.x; act[1] = a4.y; act[2] = a4.z; act[3] = a4.w;
#pragma unroll
                for (int i = 4; i < AGX_MAX_MOTORS; ++i) act[i] = 0.0f;
            } else {
#pragma unroll
                for (int i = 0; i < AGX_MAX_MOTORS; ++i) act[i] = (i < A) ? __ldcg(buf.actions + (size_t)env * A + i) : 0.0f;
            }
            // clip_actions, robots/base_multirotor.py:207-211
#pragma unroll
            for (int i = 0; i < AGX_MAX_MOTORS; ++i) act[i] = fminf(fmaxf(act[i], -10.0f), 10.0f);
        }
        fill_rows13(buf.root_state, env0, n_valid, tile, lane, vec_ok);
        if constexpr (COOP) {  // truncations are known before the physics: publish them now
            const bool trunc_early = valid && (steps_in + 1 > cfg.episode_len_steps);
            if (__ballot_sync(0xffffffffu, trunc_early)) {
                warp_raised = true;
                if (lane == 0) atomicMax(reset_flag, flag_tag);
            }
        }
        // the state is read from the tile only now: its 13 floats are not live across the loads' wait and the ballot above
        if (valid) s = unpack(tile + lane * 13);
        __syncwarp();
        AGX_TL(6);
        if (valid) {
            // every iteration runs the same instruction sequence, so n fused sub-steps are
            // bit-identical to n single-step launches
#pragma unroll 1
            for (int step = 0; step < cfg.physics_steps; ++step) {
                float Fx, Fy, Fz, Tx, Ty, Tz;
                // AGX_SHADOW_BEGIN(physics_substep)  -- tests/_shadow.py compiles the text between these markers for the host
                d = update_states(s);
                float ref[M];
                if (SP::controller(cfg) == AGX_CTRL_NONE) {  // update_motor_thrusts_with_forces
AGX_HP1_MOTOR_UNROLL
                    for (int i = 0; i < M; ++i) ref[i] = act[i];
                } else {
                    float wr[6];
                    controller_wrench<SP>(cfg, s, d, p.g, act, wr);
                    // f_ref = pinv(A) w   control/control_allocation.py:87-89
AGX_HP1_MOTOR_UNROLL
                    for (int i = 0; i < M; ++i) {
                        float acc = 0.0f;
AGX_HP1_MOTOR_UNROLL
                        for (int j = 0; j < 6; ++j) acc += cfg.alloc_pinv[i * 6 + j] * wr[j];
                        ref[i] = acc;
                    }
                }
AGX_HP1_MOTOR_UNROLL
                for (int i = 0; i < M; ++i) p.thrust[i] = motor_update<SP>(cfg, p.thrust[i], ref[i], p.tau_inc[i], p.tau_dec[i], p.k[i]);
                // thrust -> base-frame wrench about the COM (control_allocation.py:103-114 applied
                // link-local, IGE_env_manager.py:444-449; SURVEY Appendix B)
                float w6[6];
AGX_HP1_MOTOR_UNROLL
                for (int j = 0; j < 6; ++j) {
                    float acc = 0.0f;
AGX_HP1_MOTOR_UNROLL
                    for (int i = 0; i < M; ++i) acc += cfg.wrench_map[j * AGX_MAX_MOTORS + i] * p.thrust[i];
                    w6[j] = acc;
                }
                // simulate_drag, robots/base_multirotor.py:260-285 (body 0)
                float vbn = norm3(d.vb);
                V3 df = neg(ld3c(cfg.drag_lin1) * d.vb) + neg(ld3c(cfg.drag_lin2) * vbn * d.vb);
                V3 wabs{fabsf(d.wb.x), fabsf(d.wb.y), fabsf(d.wb.z)};
                V3 dtq = neg(ld3c(cfg.drag_ang1) * d.wb) + neg(ld3c(cfg.drag_ang2) * wabs * d.wb);
                if (buf.disturbance) {  // apply_disturbance :213-234 (draws stay in torch)
                    const float* dp = buf.disturbance + (size_t)env * 6;
                    df = df + ld3cg(dp);
                    dtq = dtq + ld3cg(dp + 3);
                }
                else if (!TASK && buf.dist_counter) {  // the same draw, in the kernel (physics-only launches: EnvManager's graph step); counter word from device memory
                    float d6[6];
                    disturbance_env((uint32_t)(cfg.env_id_offset + env), *buf.dist_counter + buf.dist_offset + (uint32_t)step, cfg.dist_prob, cfg.dist_max,
                                    (uint32_t)(cfg.dist_seed & 0xffffffffu), (uint32_t)(cfg.dist_seed >> 32), d6);
                    df = df + V3{d6[0], d6[1], d6[2]};
                    dtq = dtq + V3{d6[3], d6[4], d6[5]};
                }
                V3 com = ld3c(cfg.com);
                V3 F{w6[0] + df.x, w6[1] + df.y, w6[2] + df.z};
                V3 T = V3{w6[3], w6[4], w6[5]} + dtq + cross(neg(com), df);
                Fx = F.x; Fy = F.y; Fz = F.z; Tx = T.x; Ty = T.y; Tz = T.z;
                integrate<SP>(cfg, s, F, T);
                // AGX_SHADOW_END(physics_substep)
                // the last sub-step's wrench is stored here: held for after the loop, its six floats were live through every sub-step
                if (buf.body_wrench && step + 1 == cfg.physics_steps) {
                    float* bw = buf.body_wrench + (size_t)env * 6;
                    bw[0] = Fx; bw[1] = Fy; bw[2] = Fz; bw[3] = Tx; bw[4] = Ty; bw[5] = Tz;
                }
            }
            if (cfg.physics_steps == 0) {
                d = update_states(s);
                if (buf.body_wrench) {
                    float* bw = buf.body_wrench + (size_t)env * 6;
                    bw[0] = 0.f; bw[1] = 0.f; bw[2] = 0.f; bw[3] = 0.f; bw[4] = 0.f; bw[5] = 0.f;
                }
            }
        }

        AGX_TL(1);
        bool do_reset = false;
        int flag_pre = 0;
        // warp-uniform (consumed after the epilogue): in a partial tile the lanes may arrive here diverged, at different times; a flag
        // raised in between would give lanes of one warp different decisions below and a full-mask __any_sync only some of them reach
        if constexpr (COOP) flag_pre = __any_sync(0xffffffffu, *reinterpret_cast<volatile uint32_t*>(reset_flag) == flag_tag);
        if constexpr (TASK) {
            int steps = steps_in + 1;  // env_manager.py:429
            if (valid) {
                // ---- a16 reward + flags: position_setpoint_task.py:205-282 (stale derived) -----
                // AGX_SHADOW_BEGIN(position_task_reward)
                V3 e = quat_apply(quat_conj(d.qveh), tgt - s.x);
                float dist = norm3(e);
                float pos_reward = 3.0f * expf(-8.0f * dist * dist) + 2.0f * expf(-4.0f * dist * dist);
                float dist_reward = (20.0f - dist) / 40.0f;
                V3 ups = quat_rotate(s.q, V3{0.0f, 0.0f, 1.0f});
                float tilt = fabsf(1.0f - ups.z);
                float up_reward = 0.2f / (0.1f + tilt * tilt);
                float spin = norm3(d.wb);
                float ang_reward = (1.0f / (1.0f + spin * spin)) * 3.0f;
                float total = pos_reward + dist_reward + pos_reward * (up_reward + ang_reward);
                bool crash = dist > cfg.crash_distance;
                if (crash) total = -20.0f;
                bool trunc = steps > cfg.episode_len_steps;  // :172-174
                // AGX_SHADOW_END(position_task_reward)
                do_reset = crash || trunc;
                buf.reward[env] = total;
                buf.terminations[env] = crash ? 1 : 0;
                buf.truncations[env] = trunc ? 1 : 0;
                if (buf.reset_mask) buf.reset_mask[env] = do_reset ? 1 : 0;
            }
            bool fresh = !(cfg.flags & AGX_F_STRICT_STALE_OBS);
            // ---- a15 in-kernel reset, warp-cooperative Philox (see coop_rng_draw) -----------------
            const bool rng_reset = do_reset && (cfg.flags & AGX_F_DEVICE_RNG_RESET);
            const unsigned rmask = __ballot_sync(0xffffffffu, rng_reset);
            if (rmask) {
                const uint32_t my_ep = rng_reset ? __ldcg(buf.episode_count + env) : 0u;
                for (unsigned m = rmask; m; m &= m - 1) {
                    const int owner = __ffs(m) - 1;
                    const uint32_t ep = __shfl_sync(0xffffffffu, my_ep, owner);
                    reset_one_env<M>(cfg, buf, env0, owner, ep, lane, tile, s, p);
                    if (lane == owner) {
                        steps = 0;  // env_manager.py:301
                        fresh = true;
                    }
                }
            }
            if constexpr (!COOP) {
                if (valid) {
                    buf.sim_steps[env] = steps;
                    if (fresh) d = update_states(s);
                    make_obs(s, d, tgt, o);
                    if (buf.fresh_vel) {  // post-physics body velocities for the conditional obs patch
                        V3 vb = fresh ? d.vb : quat_rotate_inverse(s.q, s.v);
                        V3 wb = fresh ? d.wb : quat_rotate_inverse(s.q, s.w);
                        const size_t Ns = (size_t)N;
                        buf.fresh_vel[env] = vb.x; buf.fresh_vel[Ns + env] = vb.y; buf.fresh_vel[2 * Ns + env] = vb.z;
                        buf.fresh_vel[3 * Ns + env] = wb.x; buf.fresh_vel[4 * Ns + env] = wb.y; buf.fresh_vel[5 * Ns + env] = wb.z;
                    }
                }
                unsigned any = __ballot_sync(0xffffffffu, do_reset);
                if (any && lane == 0) atomicOr(buf.any_reset, 1);
            } else {
                if (valid) buf.sim_steps[env] = steps;
                if (__ballot_sync(0xffffffffu, do_reset)) {
                    flag_pre = 1;
                    if (!warp_raised && lane == 0) atomicMax(reset_flag, flag_tag);
                    warp_raised = true;
                }
                // ---- the decision: is anybody in the whole grid resetting this step? ----------------
                bool counted = false;
                int any = flag_pre;
                if (!any && __any_sync(0xffffffffu, valid && !fresh)) {  // rare: count ourselves in, then wait
                    if (lane == 0) atomicAdd(arrive_ctr, 1ull);
                    counted = true;
                    volatile uint32_t* fl = reset_flag;
                    const unsigned long long* cnt = arrive_ctr;
                    // until the flag rises, or every warp of this step has arrived (then the flag is final)
                    spin_until([&] { return *fl == flag_tag || ld_relaxed_gpu_u64(cnt) >= arrive_target; }, buf.any_reset, 3 | (int)(step_T << 4));
                    fence_acquire_gpu();  // a complete count orders every warp's raised flag before the re-read below
                    any = __any_sync(0xffffffffu, *fl == flag_tag);  // the flag is monotonic: one lane seeing it raised means it is
                }
                // ---- derived states for the observation: one common pass for resetting envs (new state)
                // and, if anybody reset, for everybody else (post-physics state) ------------------------
                const bool derived = buf.euler || buf.vehicle_orientation || buf.vehicle_linvel || buf.body_linvel || buf.body_angvel;
                // the root-state row, then the observation row, is written straight into the tile: no 13-float copy of either is
                // held in registers next to s, d and p (the register budget is full here: they were the epilogue's spills)
                float* row = tile + lane * 13;
                if (valid) {
                    if (fresh || any) {
                        if (derived) {
                            d = update_states(s);
                        } else {  // only the observation needs them: body-frame velocities
                            d.vb = quat_rotate_inverse(s.q, s.v);
                            d.wb = quat_rotate_inverse(s.q, s.w);
                        }
                    }
                    store_m<M>(buf.motor_thrust, env, p.thrust);
                    if (derived) store_derived(buf, env, d);
                    pack(s, row);
                }
                flush_rows13(buf.root_state, env0, n_valid, tile, lane, vec_ok);
                if (valid) make_obs(s, d, tgt, row);
                flush_rows13(buf.obs, env0, n_valid, tile, lane, vec_ok);
                if (lane == 0) {
                    // ONE release fence (MEMBAR.ALL.GPU), then relaxed operations: the tile's stores (and a raised flag) are visible before
                    // the arrival, the publish count and the done-counter (fence-based release; the consumers acquire).  Round 1 had
                    // __threadfence() (MEMBAR.SC + L1 invalidate) followed by st.release (a second MEMBAR): ncu r2 showed `membar` as the
                    // second largest stall of the kernel.  Nothing after it reads what another warp wrote, so it needs no acquire half
                    // (fence.acq_rel would add an L1 invalidation).
                    fence_release_gpu();
                    if (!counted) atomicAdd(arrive_ctr, 1ull);
                    // only with a consumer outside the kernel (observation gather); the address is formed here, not held in a register
                    // (or a spill slot) for the whole step
                    if (buf.publish_ctr) atomicAdd(buf.publish_ctr + (step_T & 3u), 1ull);
                    st_relaxed_gpu_u32(buf.tile_sync + n_tiles + t, flag_tag);  // this tile may start step T + 1
                }
            }
        }
        if constexpr (!(TASK && COOP)) {
            float r[13];
            if (valid) {
                store_m<M>(buf.motor_thrust, env, p.thrust);
                store_derived(buf, env, d);
                pack(s, r);
            }
            store_rows13(buf.root_state, env0, n_valid, tile, lane, r, vec_ok);
            if constexpr (TASK) store_rows13(buf.obs, env0, n_valid, tile, lane, o, vec_ok);
        }
    }
    AGX_TL(2);
    AGX_TL(3);
}

// refresh pass: update_states for all envs (+ obs).  only_if_flag: gated on any_reset[0] and the
// last-arriving block clears flag + arrival counter (so no memset node is needed per step).
__global__ void __launch_bounds__(kThreads)
hp1_refresh_kernel(const __grid_constant__ AgxHp1Config cfg, const __grid_constant__ AgxHp1Buffers buf, int only_if_flag,
                   int vec_ok) {
    __shared__ __align__(16) float tiles[kWarpsPerBlock][kTileFloats];
    __shared__ int s_flag;
    if (only_if_flag) {
        if (threadIdx.x == 0) {
            int f = *reinterpret_cast<volatile int*>(buf.any_reset);
            s_flag = f;
            __threadfence();
            int arrived = atomicAdd(buf.any_reset + 1, 1);
            if (arrived == (int)gridDim.x - 1) {  // every block has read the flag
                buf.any_reset[0] = 0;
                buf.any_reset[1] = 0;
            }
        }
        __syncthreads();
        if (s_flag == 0) return;
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float* tile = tiles[warp];
    const int N = cfg.num_envs;
    const int n_tiles = (N + 31) >> 5;
    for (int t = blockIdx.x * kWarpsPerBlock + warp; t < n_tiles; t += gridDim.x * kWarpsPerBlock) {
        const int env0 = t << 5;
        const int n_valid = min(32, N - env0);
        const int env = env0 + lane;
        float r[13], o[13];
        load_rows13(buf.root_state, env0, n_valid, tile, lane, r, vec_ok);
        if (lane < n_valid) {
            EnvState s = unpack(r);
            Derived d = update_states(s);
            store_derived(buf, env, d);
            if (buf.obs) {
                V3 tgt = buf.target_position ? ld3(buf.target_position + (size_t)env * 3) : V3{0, 0, 0};
                make_obs(s, d, tgt, o);
            }
        }
        if (buf.obs) store_rows13(buf.obs, env0, n_valid, tile, lane, o, vec_ok);
    }
}

// light variant of the refresh pass for the fused task step without materialised derived states:
// if any env reset this step, obs[:,7:13] <- fresh body velocities written by the main kernel.
__global__ void __launch_bounds__(256)
hp1_obs_patch_kernel(int N, const float* __restrict__ fresh_vel, float* __restrict__ obs, int* any_reset) {
    __shared__ int s_flag;
    if (threadIdx.x == 0) {
        int f = *reinterpret_cast<volatile int*>(any_reset);
        s_flag = f;
        __threadfence();
        int arrived = atomicAdd(any_reset + 1, 1);
        if (arrived == (int)gridDim.x - 1) {
            any_reset[0] = 0;
            any_reset[1] = 0;
        }
    }
    __syncthreads();
    if (s_flag == 0) return;
    const int env = blockIdx.x * blockDim.x + threadIdx.x;
    if (env >= N) return;
    float* o = obs + (size_t)env * 13 + 7;
#pragma unroll
    for (int j = 0; j < 6; ++j) o[j] = fresh_vel[(size_t)j * N + env];
}

// masked reset with caller-supplied uniforms (torch RNG, reference call order) or device RNG
template <int M>
__global__ void __launch_bounds__(kThreads)
hp1_reset_kernel(const __grid_constant__ AgxHp1Config cfg, const __grid_constant__ AgxHp1Buffers buf,
                 const uint8_t* __restrict__ mask, const __grid_constant__ AgxHp1ResetDraws dr, int have_draws) {
    const int env = blockIdx.x * blockDim.x + threadIdx.x;
    if (env >= cfg.num_envs || !mask[env]) return;
    EnvState s;
    EnvParams<M> p;
    load_params<M>(cfg, buf, env, p);
    if (have_draws) {
        float us[13], ubl[3], ubh[3], ug[12], um[4 * M];
#pragma unroll
        for (int j = 0; j < 13; ++j) us[j] = dr.state[(size_t)env * 13 + j];
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            ubl[j] = dr.bounds_lo ? dr.bounds_lo[(size_t)env * 3 + j] : 0.0f;
            ubh[j] = dr.bounds_hi ? dr.bounds_hi[(size_t)env * 3 + j] : 0.0f;
            ug[j] = dr.K_pos ? dr.K_pos[(size_t)env * 3 + j] : 0.0f;
            ug[3 + j] = dr.K_vel ? dr.K_vel[(size_t)env * 3 + j] : 0.0f;
            ug[6 + j] = dr.K_rot ? dr.K_rot[(size_t)env * 3 + j] : 0.0f;
            ug[9 + j] = dr.K_angvel ? dr.K_angvel[(size_t)env * 3 + j] : 0.0f;
        }
#pragma unroll
        for (int i = 0; i < M; ++i) {
            um[4 * i + 0] = dr.tau_inc[(size_t)env * M + i];
            um[4 * i + 1] = dr.tau_dec[(size_t)env * M + i];
            um[4 * i + 2] = dr.thrust[(size_t)env * M + i];
            um[4 * i + 3] = dr.k_thrust ? dr.k_thrust[(size_t)env * M + i] : 0.0f;
        }
        apply_reset<M>(cfg, us, ubl, ubh, ug, um, s, p);
    } else {
        uint32_t ep = buf.episode_count[env];
        device_rng_reset<M>(cfg, (uint32_t)(cfg.env_id_offset + env), ep, s, p);
        buf.episode_count[env] = ep + 1u;
    }
    float r[13];
    pack(s, r);
#pragma unroll
    for (int j = 0; j < 13; ++j) buf.root_state[(size_t)env * 13 + j] = r[j];
    store_m<M>(buf.motor_thrust, env, p.thrust);
    store_reset_params<M>(buf, env, p);
    if (buf.sim_steps) buf.sim_steps[env] = 0;  // env_manager.py:301
}

int validate(const AgxHp1Config* cfg, const AgxHp1Buffers* buf, bool task) {
    if (!cfg || !buf) return agx_set_error(AGX_E_NULL, "cfg/buf is NULL");
    if (cfg->num_envs < 0) return agx_set_error(AGX_E_INVALID, "num_envs < 0");
    if (cfg->num_motors != 4 && cfg->num_motors != 8)
        return agx_set_error(AGX_E_INVALID, "num_motors must be 4 or 8 (got %d)", cfg->num_motors);
    if (cfg->controller < AGX_CTRL_NONE || cfg->controller > AGX_CTRL_VELOCITY_STEERING)
        return agx_set_error(AGX_E_INVALID, "unknown controller id %d", cfg->controller);
    int need = (cfg->controller == AGX_CTRL_NONE) ? cfg->num_motors : (cfg->controller == AGX_CTRL_FULLY_ACTUATED ? 7 : 4);
    if (cfg->num_actions != need)
        return agx_set_error(AGX_E_INVALID, "controller %d needs %d action columns (got %d)", cfg->controller, need, cfg->num_actions);
    if (cfg->physics_steps < 0) return agx_set_error(AGX_E_INVALID, "physics_steps < 0");
    if (cfg->num_envs == 0) return AGX_OK;  /* empty batch: nothing to check or launch */
    if (!buf->root_state || !buf->motor_thrust || !buf->actions) return agx_set_error(AGX_E_NULL, "root_state/motor_thrust/actions is NULL");
    if (((uintptr_t)buf->motor_thrust | (uintptr_t)buf->actions | (uintptr_t)buf->tau_inc | (uintptr_t)buf->tau_dec |
         (uintptr_t)buf->k_thrust | (uintptr_t)buf->vehicle_orientation) & 15)
        return agx_set_error(AGX_E_INVALID, "[N,M]/[N,4] arrays must be 16-byte aligned");
    if (task) {
        if (!buf->sim_steps || !buf->obs || !buf->reward || !buf->terminations || !buf->truncations || !buf->any_reset)
            return agx_set_error(AGX_E_NULL, "task step needs sim_steps/obs/reward/terminations/truncations/any_reset");
        if ((cfg->flags & AGX_F_DEVICE_RNG_RESET) && !buf->episode_count)
            return agx_set_error(AGX_E_NULL, "device-RNG reset needs episode_count");
    }
    return AGX_OK;
}

inline int vec_ok_of(const AgxHp1Buffers* buf) {
    return (((uintptr_t)buf->root_state | (uintptr_t)buf->obs) & 15) == 0;
}
// ---- instantiation table ------------------------------------------------------------------------------------------------
// The single-launch task kernel and the physics-only kernel exist in a generic form (every switch read at run time) and in forms
// specialised (HpSpec) for the controller x motor-model combinations the shipped robots use; a launch picks the match.
#define AGX_SPEC_FLAGS_ALL (AGX_F_USE_RPS | AGX_F_MOTOR_RK4 | AGX_F_DISCRETE_MIX | AGX_F_GYROSCOPIC)
#ifndef AGX_HP1_NO_SPEC
#define AGX_HP1_SPEC_LIST(X)                                                                                      \
    X(4, AGX_CTRL_ATTITUDE, AGX_SPEC_FLAGS_ALL)      /* base_quadrotor + lee_attitude_control (position task, BASELINE configs[1]) */ \
    X(4, AGX_CTRL_VELOCITY, AGX_SPEC_FLAGS_ALL)      /* lmf2 / base_quadrotor velocity control (navigation tasks) */      \
    X(4, AGX_CTRL_POSITION, AGX_SPEC_FLAGS_ALL)                                                                   \
    X(4, AGX_CTRL_ACCELERATION, AGX_SPEC_FLAGS_ALL)                                                               \
    X(4, AGX_CTRL_NONE, AGX_SPEC_FLAGS_ALL)          /* motor-command tasks */                                     \
    X(8, AGX_CTRL_FULLY_ACTUATED, (AGX_F_MOTOR_RK4 | AGX_F_DISCRETE_MIX | AGX_F_GYROSCOPIC)) /* base_octarotor / ROV */ \
    X(8, AGX_CTRL_VELOCITY, (AGX_F_MOTOR_RK4 | AGX_F_DISCRETE_MIX | AGX_F_GYROSCOPIC))
#else
#define AGX_HP1_SPEC_LIST(X)
#endif

using StepKernel = void (*)(const AgxHp1Config, const AgxHp1Buffers, int, uint32_t);
template <bool TASK, bool COOP>
StepKernel pick_kernel(const AgxHp1Config* cfg) {
    const int id = hp_spec_id(cfg->controller, cfg->flags);
#define AGX_X(M_, C_, F_) \
    if (cfg->num_motors == M_ && id == hp_spec_id(C_, F_)) return hp1_step_kernel<M_, TASK, COOP, hp_spec_id(C_, F_)>;
    AGX_HP1_SPEC_LIST(AGX_X)
#undef AGX_X
    return cfg->num_motors == 4 ? hp1_step_kernel<4, TASK, COOP, -1> : hp1_step_kernel<8, TASK, COOP, -1>;
}

// how many CTAs of the single-launch task kernel can be co-resident on this device (cached per kernel)
inline int coop_capacity(StepKernel k) {
    static StepKernel seen[32];
    static int caps[32], n_seen = 0;
    for (int i = 0; i < n_seen; ++i)
        if (seen[i] == k) return caps[i];
    int dev = 0, sms = 0, per_sm = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    agx_set_coresident_carveout(k);  // same shared-memory carve-out as the gather kernels that run beside this one (agx_common.cuh)
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k, kThreads, 0);
    const int cap = sms * per_sm;
    if (n_seen < 32) { seen[n_seen] = k; caps[n_seen] = cap; ++n_seen; }
    return cap;
}
// CTA slots kept free for kernels that run BESIDE the chained step (the observation gather's push kernel): the one-sided grid
// barrier needs every CTA of a step resident, so the step only takes the single-launch path when it fits with this margin.
// What liveness needs is one slot per ring slot, for the one-warp ready gates (tests/_protocol_model.py): a push CTA only becomes
// resident after its ready gate has seen the step published, so the push CTAs themselves (256 threads each: 24 of them take the
// threads of 96 step CTAs) need not fit beside the step.  32 is that bound for a ring of 4 plus margin; the margin is not measured on
// multi-GPU H100s.  H100: 132 SMs x 8 = 1056 slots - 32 = 1024 = exactly the grid of 65,536 envs.  Any loss of occupancy or fewer
// SMs moves that size to the two-launch path (slower; same results except roll / yaw after a reset, DESIGN §6 Checks): bench.py's config5_env_sweep reports the path per size.
#ifndef AGX_HP1_COOP_RESERVE
#define AGX_HP1_COOP_RESERVE 32
#endif
constexpr int kCoopReserve = AGX_HP1_COOP_RESERVE;
inline int grid_for(int n_envs) {
    int tiles = (n_envs + 31) / 32;
    int blocks = (tiles + kWarpsPerBlock - 1) / kWarpsPerBlock;
    return blocks < 1 ? 1 : blocks;
}

// does the fused task step of (cfg, buf) take the single-launch, per-tile chained path?
inline bool hp1_task_step_is_chained(const AgxHp1Config* cfg, const AgxHp1Buffers* buf) {
    const bool strict_fused = (cfg->flags & AGX_F_DEVICE_RNG_RESET) && (cfg->flags & AGX_F_STRICT_STALE_OBS);
    return strict_fused && buf->tile_sync && coop_capacity(pick_kernel<true, true>(cfg)) - kCoopReserve >= grid_for(cfg->num_envs);
}

// The chained kernel of the task step and whether it is taken, resolved once per shape of (cfg, buf): the flagship enqueues a step every
// few microseconds, each from the same shape.  Only the shape is remembered; every launch passes the caller's live cfg and buf.
struct TaskPlan {
    int num_envs = -1, num_motors = 0, controller = 0, flags = 0;
    bool tile_sync = false, chained = false;
    StepKernel coop = nullptr;
};
inline const TaskPlan& task_plan(const AgxHp1Config* cfg, const AgxHp1Buffers* buf) {
    thread_local TaskPlan p;
    if (p.num_envs != cfg->num_envs || p.num_motors != cfg->num_motors || p.controller != cfg->controller || p.flags != cfg->flags ||
        p.tile_sync != (buf->tile_sync != nullptr)) {
        p.num_envs = cfg->num_envs; p.num_motors = cfg->num_motors; p.controller = cfg->controller; p.flags = cfg->flags;
        p.tile_sync = buf->tile_sync != nullptr;
        p.coop = pick_kernel<true, true>(cfg);
        p.chained = hp1_task_step_is_chained(cfg, buf);
    }
    return p;
}
cudaLaunchAttribute* chained_attr() {
    static cudaLaunchAttribute a = [] {
        cudaLaunchAttribute x = {};
        x.id = cudaLaunchAttributeProgrammaticStreamSerialization;
        x.val.programmaticStreamSerializationAllowed = 1;
        return x;
    }();
    return &a;
}

// the fused task step; step = T of a chained launch, or kClaimOnDevice
int task_step(const AgxHp1Config* cfg, const AgxHp1Buffers* buf, void* stream, void* ev_after_main, uint32_t step) {
    int rc = validate(cfg, buf, true);
    if (rc) return rc;
    if (cfg->num_envs == 0) return AGX_OK;
    cudaStream_t st = (cudaStream_t)stream;
    int g = grid_for(cfg->num_envs), v = vec_ok_of(buf);
    const TaskPlan& plan = task_plan(cfg, buf);
    if (plan.chained && !ev_after_main) {
        // single launch: the whole grid is resident at once (g <= occupancy x SMs), so the in-kernel
        // one-sided barrier cannot starve -- no cooperative-launch API needed for that
        cudaLaunchConfig_t lc = {};
        lc.gridDim = dim3(g);
        lc.blockDim = dim3(kThreads);
        lc.stream = st;
        lc.attrs = chained_attr();
        lc.numAttrs = 1;
        cudaError_t e = cudaLaunchKernelEx(&lc, plan.coop, *cfg, *buf, v, step);
        return agx_check_cuda(e, "hp1_step_kernel<task, single-launch>");
    }
    const bool strict_fused = (cfg->flags & AGX_F_DEVICE_RNG_RESET) && (cfg->flags & AGX_F_STRICT_STALE_OBS);
    const bool derived = buf->euler || buf->vehicle_orientation || buf->vehicle_linvel || buf->body_linvel || buf->body_angvel;
    pick_kernel<true, false>(cfg)<<<g, kThreads, 0, st>>>(*cfg, *buf, v, 0u);
    rc = agx_check_launch("hp1_step_kernel<task>");
    if (rc) return rc;
    if (ev_after_main) {
        rc = agx_check_cuda(cudaEventRecord((cudaEvent_t)ev_after_main, st), "cudaEventRecord");
        if (rc) return rc;
    }
    // stale-derived-state quirk (SURVEY 3.1): if ANY env reset this step the reference refreshes
    // the derived states of ALL envs before the observation is read (base_multirotor.py:204-205).
    if (strict_fused) {
        if (buf->fresh_vel && !derived) {
            hp1_obs_patch_kernel<<<(cfg->num_envs + 255) / 256, 256, 0, st>>>(cfg->num_envs, buf->fresh_vel, buf->obs, buf->any_reset);
            rc = agx_check_launch("hp1_obs_patch_kernel");
        } else {
            hp1_refresh_kernel<<<g, kThreads, 0, st>>>(*cfg, *buf, 1, v);
            rc = agx_check_launch("hp1_refresh_kernel");
        }
    }
    return rc;
}

}  // namespace

extern "C" {

int agx_hp1_task_step_is_chained(const AgxHp1Config* cfg, const AgxHp1Buffers* buf) {
    if (!cfg || !buf) return agx_set_error(AGX_E_NULL, "cfg/buf is NULL");
    if (cfg->num_motors != 4 && cfg->num_motors != 8) return agx_set_error(AGX_E_INVALID, "num_motors must be 4 or 8");
    return hp1_task_step_is_chained(cfg, buf) ? 1 : 0;
}

__global__ void counter_add_kernel(uint32_t* c, uint32_t n) { *c += n; }
int agx_counter_add(uint32_t* counter, uint32_t n, void* stream) {
    if (!counter) return agx_set_error(AGX_E_NULL, "agx_counter_add: NULL counter");
    counter_add_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(counter, n);
    return agx_check_launch("counter_add_kernel");
}

int agx_set_spin_timeout_ms(uint64_t ms) {
    const unsigned long long ns = (unsigned long long)ms * 1000000ull;
    int rc = agx_check_cuda(cudaMemcpyToSymbol(g_hp1_spin_timeout_ns, &ns, sizeof(ns)), "agx_set_spin_timeout_ms");
    return rc ? rc : agx_obs_gather_set_timeout_ns(ns);
}

// error word of the chained step's bounded waits (any_reset[2]); synchronises the stream
int agx_hp1_check(const AgxHp1Buffers* buf, void* stream) {
    if (!buf || !buf->any_reset) return agx_set_error(AGX_E_NULL, "buf/any_reset is NULL");
    int32_t w = 0;
    int rc = agx_check_cuda(cudaMemcpyAsync(&w, buf->any_reset + kErrWord, sizeof(w), cudaMemcpyDeviceToHost, (cudaStream_t)stream), "agx_hp1_check");
    if (rc) return rc;
    rc = agx_check_cuda(cudaStreamSynchronize((cudaStream_t)stream), "agx_hp1_check");
    if (rc) return rc;
    return w ? agx_set_error(AGX_E_TIMEOUT, "a chained-step wait timed out (error word %d): the step kernel was not fully resident "
                                            "or a producer never arrived", w) : AGX_OK;
}

#ifdef AGX_TIMELINE
int agx_dbg_timeline(unsigned long long* host_out) {
    return agx_check_cuda(cudaMemcpyFromSymbol(host_out, g_timeline, sizeof(g_timeline)), "timeline");
}
__global__ void dbg_empty_full_params(const __grid_constant__ AgxHp1Config, const __grid_constant__ AgxHp1Buffers, int, uint32_t) {}
__global__ void dbg_empty_buf_params(const __grid_constant__ AgxHp1Buffers) {}
// host microseconds per call, n calls each: out[0] the task-step entry up to its launch (validation, plan), out[1] cudaLaunchKernelEx
// of an empty kernel with the chained step's launch configuration and parameter block, out[2] the same with AgxHp1Buffers alone
int agx_dbg_host_costs(const AgxHp1Config* cfg, const AgxHp1Buffers* buf, void* stream, int n, double* out) {
    using clk = std::chrono::steady_clock;
    const auto us = [n](clk::time_point a, clk::time_point b) { return std::chrono::duration<double, std::micro>(b - a).count() / n; };
    volatile int sink = 0;
    auto t0 = clk::now();
    for (int i = 0; i < n; ++i) {
        int rc = validate(cfg, buf, true);
        sink = sink + rc + (int)task_plan(cfg, buf).chained + grid_for(cfg->num_envs) + vec_ok_of(buf);
    }
    auto t1 = clk::now();
    cudaLaunchConfig_t lc = {};
    lc.gridDim = dim3(grid_for(cfg->num_envs));
    lc.blockDim = dim3(kThreads);
    lc.stream = (cudaStream_t)stream;
    lc.attrs = chained_attr();
    lc.numAttrs = 1;
    for (int i = 0; i < n; ++i) cudaLaunchKernelEx(&lc, dbg_empty_full_params, *cfg, *buf, 1, (uint32_t)i);
    auto t2 = clk::now();
    for (int i = 0; i < n; ++i) cudaLaunchKernelEx(&lc, dbg_empty_buf_params, *buf);
    auto t3 = clk::now();
    out[0] = us(t0, t1); out[1] = us(t1, t2); out[2] = us(t2, t3);
    return agx_check_cuda(cudaStreamSynchronize((cudaStream_t)stream), "agx_dbg_host_costs");
}
#endif

int agx_hp1_physics_step(const AgxHp1Config* cfg, const AgxHp1Buffers* buf, void* stream) {
    int rc = validate(cfg, buf, false);
    if (rc) return rc;
    if (cfg->num_envs == 0) return AGX_OK;
    cudaStream_t st = (cudaStream_t)stream;
    int g = grid_for(cfg->num_envs), v = vec_ok_of(buf);
    pick_kernel<false, false>(cfg)<<<g, kThreads, 0, st>>>(*cfg, *buf, v, 0u);
    return agx_check_launch("hp1_step_kernel");
}

int agx_hp1_position_task_step(const AgxHp1Config* cfg, const AgxHp1Buffers* buf, void* stream) {
    return agx_hp1_position_task_step_profiled(cfg, buf, stream, nullptr);
}

int agx_hp1_position_task_step_gathered(const AgxHp1Config* cfg, const AgxHp1Buffers* buf, void* stream, const uint32_t* gate_read_done,
                                        uint32_t gate_need_epoch, uint32_t* gate_error_word, const AgxObsGatherPush* push, void* push_stream) {
    int rc = AGX_OK;
    if (gate_read_done) rc = agx_obs_gather_gate(gate_read_done, gate_need_epoch, gate_error_word, stream);
    if (rc == AGX_OK) rc = agx_hp1_position_task_step_profiled(cfg, buf, stream, nullptr);
    if (rc == AGX_OK && push) rc = agx_obs_gather_push(push, push_stream);
    return rc;
}

int agx_hp1_position_task_step_profiled(const AgxHp1Config* cfg, const AgxHp1Buffers* buf, void* stream,
                                        void* ev_after_main) {
    return task_step(cfg, buf, stream, ev_after_main, kClaimOnDevice);
}

int agx_hp1_position_task_step_at(const AgxHp1Config* cfg, const AgxHp1Buffers* buf, void* stream, uint32_t step_index) {
    if (step_index == kClaimOnDevice) return agx_set_error(AGX_E_INVALID, "step_index 0xffffffff is reserved");
    return task_step(cfg, buf, stream, nullptr, step_index);
}

int agx_hp1_reset(const AgxHp1Config* cfg, const AgxHp1Buffers* buf, const uint8_t* mask, const AgxHp1ResetDraws* draws,
                  void* stream) {
    if (cfg && cfg->num_envs == 0) return AGX_OK;
    if (!cfg || !buf || !mask) return agx_set_error(AGX_E_NULL, "cfg/buf/mask is NULL");
    if (cfg->num_motors != 4 && cfg->num_motors != 8) return agx_set_error(AGX_E_INVALID, "num_motors must be 4 or 8");
    if (!buf->root_state || !buf->motor_thrust) return agx_set_error(AGX_E_NULL, "root_state/motor_thrust is NULL");
    if (draws) {
        if (!draws->state || !draws->tau_inc || !draws->tau_dec || !draws->thrust)
            return agx_set_error(AGX_E_NULL, "reset draws need state/tau_inc/tau_dec/thrust");
        if ((cfg->flags & AGX_F_USE_RPS) && !draws->k_thrust) return agx_set_error(AGX_E_NULL, "use_rps reset needs k_thrust draws");
        if ((cfg->flags & AGX_F_RANDOMIZE_GAINS) && !(draws->K_pos && draws->K_vel && draws->K_rot && draws->K_angvel))
            return agx_set_error(AGX_E_NULL, "randomised gains need K_* draws");
    } else if (!buf->episode_count) {
        return agx_set_error(AGX_E_NULL, "device-RNG reset needs episode_count");
    }
    if (cfg->num_envs == 0) return AGX_OK;
    cudaStream_t st = (cudaStream_t)stream;
    AgxHp1ResetDraws d0 = {};
    const AgxHp1ResetDraws& d = draws ? *draws : d0;
    int threads = kThreads, g = (cfg->num_envs + threads - 1) / threads;
    if (cfg->num_motors == 4) hp1_reset_kernel<4><<<g, threads, 0, st>>>(*cfg, *buf, mask, d, draws != nullptr);
    else hp1_reset_kernel<8><<<g, threads, 0, st>>>(*cfg, *buf, mask, d, draws != nullptr);
    return agx_check_launch("hp1_reset_kernel");
}

int agx_hp1_refresh(const AgxHp1Config* cfg, const AgxHp1Buffers* buf, int only_if_flag, void* stream) {
    if (cfg && cfg->num_envs == 0) return AGX_OK;
    if (!cfg || !buf) return agx_set_error(AGX_E_NULL, "cfg/buf is NULL");
    if (!buf->root_state) return agx_set_error(AGX_E_NULL, "root_state is NULL");
    if (only_if_flag && !buf->any_reset) return agx_set_error(AGX_E_NULL, "only_if_flag needs any_reset");
    if (cfg->num_envs == 0) return AGX_OK;
    hp1_refresh_kernel<<<grid_for(cfg->num_envs), kThreads, 0, (cudaStream_t)stream>>>(*cfg, *buf, only_if_flag, vec_ok_of(buf));
    return agx_check_launch("hp1_refresh_kernel");
}

}  // extern "C"
