// Observation all-gather as a single kernel of NVLink peer stores + flag handshake (H100 / NVSwitch:
// every peer is reachable at full bandwidth, so each rank simply writes its shard into every
// peer's buffer).  Used instead of an NCCL collective on the step path, where a step is too short to hide an NCCL launch.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/aerial_gym_b200.h"
#include "agx_common.cuh"

namespace {

__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

__device__ __forceinline__ unsigned long long gt_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

struct PeerTable {
    float4* buf[AGX_MAX_PEERS];
    uint32_t* flag[AGX_MAX_PEERS];
};

__global__ void __launch_bounds__(256)
p2p_allgather_kernel(const float4* __restrict__ local, void* const* __restrict__ peer_bufs, uint32_t* const* __restrict__ peer_flags,
                     int world, int rank, size_t n_vec, uint32_t epoch, uint32_t* scratch) {
    __shared__ PeerTable t;
    if (threadIdx.x < world) {
        t.buf[threadIdx.x] = reinterpret_cast<float4*>(peer_bufs[threadIdx.x]) + (size_t)rank * n_vec;
        t.flag[threadIdx.x] = peer_flags[threadIdx.x];
    }
    __syncthreads();
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_vec; i += (size_t)gridDim.x * blockDim.x) {
        float4 v = local[i];
        for (int p = 0; p < world; ++p) t.buf[p][i] = v;  // own slot too: the gathered buffer is complete locally
    }
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned done = atomicAdd(scratch, 1u);
        if (done == gridDim.x - 1) {  // all blocks of this rank have stored + fenced
            *scratch = 0u;
            __threadfence_system();
            for (int p = 0; p < world; ++p) st_release_sys(t.flag[p] + rank, epoch);
            // wait until every peer has published this epoch into OUR flag words
            const uint32_t* mine = t.flag[rank];
            for (int q = 0; q < world; ++q) {
                const unsigned long long t0 = gt_ns();
                unsigned polls = 0;
                while ((int32_t)(ld_acquire_sys(mine + q) - epoch) < 0) {
                    // a missing peer must not hang the GPU forever, and a late one must not kill the context: wall-clock bound, no trap
                    if ((++polls & 255u) == 0u && gt_ns() - t0 > 20ull * 1000ull * 1000ull * 1000ull) break;
                }
            }
        }
    }
}

// ---- pipelined form: push (sender) / wait (receiver) ------------------------------------------------------------------
__device__ unsigned long long g_gather_spin_timeout_ns = 20ull * 1000ull * 1000ull * 1000ull;
__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ unsigned long long ld_acquire_gpu_u64(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
// wall-clock bounded wait; on expiry: error word, no trap (see hp1.cu spin_until)
// error word: (epoch << 8) | code, code 1 = a push never saw its producer step complete, 2 = a wait never saw a peer's flag
template <class Pred>
__device__ __forceinline__ bool spin_until(Pred ok, uint32_t* err_word, uint32_t code) {
    if (ok()) return true;
    volatile uint32_t* err = err_word;
    if (*err) return false;
    const long long t0 = clock64();
    const long long limit = (long long)g_gather_spin_timeout_ns * 2;  // ns -> SM cycles at <= 2 GHz; clock64 is monotonic per SM (%globaltimer may be re-synchronised and jump)
    unsigned polls = 0;
    while (!ok()) {
        if ((++polls & 63u) == 0u) {
            if (*err) return false;
            if (clock64() - t0 > limit) {
                atomicCAS(err_word, 0u, code);
                return false;
            }
        }
        __nanosleep(64);
    }
    return true;
}

// one 16-byte store to the NVSwitch multicast address: the switch writes it into every rank's copy of the buffer
__device__ __forceinline__ void multimem_st_f4(float4* mc, float4 v) {
    asm volatile("multimem.st.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(mc), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

constexpr int kPushThreads = 256;
constexpr int kPushUnroll = 4;

// <= 32 registers: one push CTA fits beside seven 128-register step CTAs on an SM
__global__ void __launch_bounds__(kPushThreads, 8)
obs_gather_push_kernel(const __grid_constant__ AgxObsGatherPush a, size_t n_vec) {
    __shared__ float4* s_dst[AGX_MAX_PEERS];
    __shared__ int s_npeer;
    const float4* __restrict__ local = reinterpret_cast<const float4*>(a.local);
    if (threadIdx.x == 0) {
        int n = 0;
        // peers in a rank-dependent rotation: at any moment the ranks store to different destinations
        for (int k = 1; k <= a.world; ++k) {
            const int p = (a.rank + k) % a.world;
            float4* dst = reinterpret_cast<float4*>(a.peer_bufs[p]) + (size_t)a.rank * n_vec;
            if (dst == local) continue;  // the step wrote its observation straight into the own slot
            s_dst[n++] = dst;
        }
        s_npeer = n;
        if (a.ready_ctr) {
            const unsigned long long* c = a.ready_ctr;
            const unsigned long long want = a.ready_target;
            spin_until([&] { return ld_acquire_gpu_u64(c) >= want; }, a.error_word, (a.epoch << 8) | 1u);
        }
    }
    __syncthreads();
    const int np = s_npeer;
    const size_t stride = (size_t)gridDim.x * kPushThreads;
    size_t i = (size_t)blockIdx.x * kPushThreads + threadIdx.x;
    if (a.mc_buf) {  // NVSwitch multicast: one store per 16 bytes, whatever the world size (this rank's own copy is rewritten with the same bytes)
        float4* mc = reinterpret_cast<float4*>(a.mc_buf) + (size_t)a.rank * n_vec;
        for (; i + (kPushUnroll - 1) * stride < n_vec; i += kPushUnroll * stride) {
            float4 v[kPushUnroll];
#pragma unroll
            for (int u = 0; u < kPushUnroll; ++u) v[u] = __ldcg(local + i + u * stride);
#pragma unroll
            for (int u = 0; u < kPushUnroll; ++u) multimem_st_f4(mc + i + u * stride, v[u]);
        }
        for (; i < n_vec; i += stride) multimem_st_f4(mc + i, __ldcg(local + i));
        i = n_vec;  // nothing left for the unicast loops
    }
    for (; i + (kPushUnroll - 1) * stride < n_vec; i += kPushUnroll * stride) {
        float4 v[kPushUnroll];
#pragma unroll
        for (int u = 0; u < kPushUnroll; ++u) v[u] = __ldcg(local + i + u * stride);  // L2: never a stale L1 line of an earlier step
        for (int p = 0; p < np; ++p) {
            float4* d = s_dst[p];
#pragma unroll
            for (int u = 0; u < kPushUnroll; ++u) d[i + u * stride] = v[u];
        }
    }
    for (; i < n_vec; i += stride) {
        const float4 v = __ldcg(local + i);
        for (int p = 0; p < np; ++p) s_dst[p][i] = v;
    }
    __syncthreads();  // the CTA's loads have returned (their values went into the stores) and its peer stores are ordered before thread 0's fences
    if (threadIdx.x == 0) {
        if (a.read_done && atomicAdd(a.scratch + 1, 1u) == gridDim.x - 1) {  // every CTA has finished READING `local`:
            a.scratch[1] = 0u;                                               // the producer may overwrite it (agx_obs_gather_gate)
            asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(a.read_done), "r"(a.epoch) : "memory");
        }
        __threadfence_system();  // waits until this CTA's NVLink stores have been performed
        if (atomicAdd(a.scratch, 1u) == gridDim.x - 1) {  // ... and so have everybody else's
            a.scratch[0] = 0u;
            __threadfence_system();
            for (int p = 0; p < a.world; ++p) st_release_sys(a.peer_flags[p] + a.flag_slot * AGX_MAX_PEERS + a.rank, a.epoch);
        }
    }
}

// gate in front of a chained step: launched with programmatic stream serialization BETWEEN two step launches, it lets the next
// launch in (griddepcontrol.launch_dependents) only when the push that last read the ring slot has finished reading.  One warp, no
// resources to speak of: while it waits, the step behind it is not resident, so the push it waits for always finds CTA slots.
__global__ void __launch_bounds__(32)
obs_gather_gate_kernel(const uint32_t* __restrict__ read_done, uint32_t need_epoch, uint32_t* error_word) {
    if (threadIdx.x == 0) {
        spin_until([&] {
            uint32_t v;
            asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(read_done) : "memory");
            return (int32_t)(v - need_epoch) >= 0;
        }, error_word, (need_epoch << 8) | 3u);
    }
    __syncwarp();
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}

// "ready" gate on the push's own stream: ONE warp waits for the producer step's published-tile counter, then lets the push kernel
// behind it in (programmatic stream serialization).  The push's CTAs are therefore never resident while they would only wait: beside
// a step that needs its whole grid co-resident there are at most a few one-warp gates, not 96 spinning 256-thread CTAs.
__global__ void __launch_bounds__(32)
obs_gather_ready_kernel(const unsigned long long* __restrict__ ready_ctr, unsigned long long ready_target, uint32_t* error_word, uint32_t epoch) {
    if (threadIdx.x == 0) spin_until([&] { return ld_acquire_gpu_u64(ready_ctr) >= ready_target; }, error_word, (epoch << 8) | 1u);
    __syncwarp();
    __threadfence();
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}

__global__ void __launch_bounds__(32)
obs_gather_wait_kernel(const uint32_t* __restrict__ my_flags, int world, uint32_t epoch, uint32_t* error_word) {
    const int q = threadIdx.x;
    if (q < world) spin_until([&] { return (int32_t)(ld_acquire_sys(my_flags + q) - epoch) >= 0; }, error_word, (epoch << 8) | ((uint32_t)q << 4) | 2u);
    __syncwarp();
    __threadfence_system();
}

}  // namespace

extern "C" int agx_obs_gather_set_timeout_ns(uint64_t ns) {
    const unsigned long long v = ns;
    return agx_check_cuda(cudaMemcpyToSymbol(g_gather_spin_timeout_ns, &v, sizeof(v)), "agx_obs_gather_set_timeout_ns");
}

extern "C" int agx_obs_gather_push(const AgxObsGatherPush* a, void* stream) {
    if (!a || !a->local || !a->peer_bufs || !a->peer_flags || !a->scratch || !a->error_word)
        return agx_set_error(AGX_E_NULL, "obs_gather_push: NULL argument");
    if (a->world < 1 || a->world > AGX_MAX_PEERS || a->rank < 0 || a->rank >= a->world)
        return agx_set_error(AGX_E_INVALID, "obs_gather_push: bad world/rank");
    if (a->bytes % 16 || ((uintptr_t)a->local & 15)) return agx_set_error(AGX_E_INVALID, "obs_gather_push: bytes and local must be 16-byte aligned");
    if (a->epoch == 0) return agx_set_error(AGX_E_INVALID, "obs_gather_push: epoch starts at 1");
    if ((uintptr_t)a->ready_ctr & 7) return agx_set_error(AGX_E_INVALID, "obs_gather_push: ready_ctr must be 8-byte aligned");
    if (a->flag_slot < 0 || a->flag_slot > 3) return agx_set_error(AGX_E_INVALID, "obs_gather_push: flag_slot must be in [0, 3]");
    if (a->bytes == 0) return AGX_OK;
    const size_t n_vec = a->bytes / 16;
    long long ctas = (long long)((n_vec + (size_t)kPushThreads * kPushUnroll - 1) / ((size_t)kPushThreads * kPushUnroll));
    const int cap = a->max_ctas > 0 ? a->max_ctas : 24;
    if (ctas > cap) ctas = cap;
    if (ctas < 1) ctas = 1;
    static bool carve_set = false;
    if (!carve_set) {  // same shared-memory carve-out as the step kernel it runs beside (hp1.cu coop_capacity)
        agx_set_coresident_carveout(obs_gather_push_kernel);
        agx_set_coresident_carveout(obs_gather_wait_kernel);
        carve_set = true;
    }
    if (a->ready_ctr) {
        // one-warp gate first, the push itself as its programmatic dependent with nothing left to wait for
        static bool gate_carve = false;
        if (!gate_carve) {
            agx_set_coresident_carveout(obs_gather_ready_kernel);
            gate_carve = true;
        }
        obs_gather_ready_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(a->ready_ctr, a->ready_target, a->error_word, a->epoch);
        int rc = agx_check_launch("obs_gather_ready_kernel");
        if (rc) return rc;
        AgxObsGatherPush b = *a;
        b.ready_ctr = nullptr;
        cudaLaunchConfig_t lc = {};
        lc.gridDim = dim3((unsigned)ctas);
        lc.blockDim = dim3(kPushThreads);
        lc.stream = (cudaStream_t)stream;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        at[0].val.programmaticStreamSerializationAllowed = 1;
        lc.attrs = at;
        lc.numAttrs = 1;
        return agx_check_cuda(cudaLaunchKernelEx(&lc, obs_gather_push_kernel, b, n_vec), "obs_gather_push_kernel");
    }
    obs_gather_push_kernel<<<(int)ctas, kPushThreads, 0, (cudaStream_t)stream>>>(*a, n_vec);
    return agx_check_launch("obs_gather_push_kernel");
}

extern "C" int agx_obs_gather_gate(const uint32_t* read_done, uint32_t need_epoch, uint32_t* error_word, void* stream) {
    if (!read_done || !error_word) return agx_set_error(AGX_E_NULL, "obs_gather_gate: NULL argument");
    static bool carve_set = false;
    if (!carve_set) {
        agx_set_coresident_carveout(obs_gather_gate_kernel);
        carve_set = true;
    }
    cudaLaunchConfig_t lc = {};
    lc.gridDim = dim3(1);
    lc.blockDim = dim3(32);
    lc.stream = (cudaStream_t)stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    lc.attrs = at;
    lc.numAttrs = 1;
    return agx_check_cuda(cudaLaunchKernelEx(&lc, obs_gather_gate_kernel, read_done, need_epoch, error_word), "obs_gather_gate_kernel");
}

extern "C" int agx_obs_gather_wait(const uint32_t* my_flags, int flag_slot, int world, uint32_t epoch, uint32_t* error_word, void* stream) {
    if (!my_flags || !error_word) return agx_set_error(AGX_E_NULL, "obs_gather_wait: NULL argument");
    if (world < 1 || world > AGX_MAX_PEERS || flag_slot < 0 || flag_slot > 3) return agx_set_error(AGX_E_INVALID, "obs_gather_wait: bad world / flag_slot");
    static bool carve_set = false;
    if (!carve_set) {
        agx_set_coresident_carveout(obs_gather_wait_kernel);
        carve_set = true;
    }
    obs_gather_wait_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(my_flags + flag_slot * AGX_MAX_PEERS, world, epoch, error_word);
    return agx_check_launch("obs_gather_wait_kernel");
}

extern "C" int agx_obs_gather_check(const uint32_t* error_word, void* stream) {
    if (!error_word) return agx_set_error(AGX_E_NULL, "obs_gather_check: NULL argument");
    uint32_t w = 0;
    int rc = agx_check_cuda(cudaMemcpyAsync(&w, error_word, sizeof(w), cudaMemcpyDeviceToHost, (cudaStream_t)stream), "agx_obs_gather_check");
    if (rc) return rc;
    rc = agx_check_cuda(cudaStreamSynchronize((cudaStream_t)stream), "agx_obs_gather_check");
    if (rc) return rc;
    if (!w) return AGX_OK;
    if ((w & 15u) == 3u) return agx_set_error(AGX_E_TIMEOUT, "observation gather: the gate in front of a step never saw the push of epoch %u finish reading (wait timed out)", w >> 8);
    return (w & 15u) == 1u ? agx_set_error(AGX_E_TIMEOUT, "observation gather: the push of epoch %u never saw its producer step complete (wait timed out)", w >> 8)
                           : agx_set_error(AGX_E_TIMEOUT, "observation gather: the wait for epoch %u never saw rank %u's flag (wait timed out)", w >> 8, (w >> 4) & 15u);
}

extern "C" int agx_p2p_allgather(const void* local, void* const* peer_bufs, uint32_t* const* peer_flags, int world, int rank,
                                 uint64_t bytes, uint32_t epoch, uint32_t* scratch, void* stream) {
    if (!local || !peer_bufs || !peer_flags || !scratch) return agx_set_error(AGX_E_NULL, "p2p_allgather: NULL argument");
    if (world < 1 || world > AGX_MAX_PEERS || rank < 0 || rank >= world) return agx_set_error(AGX_E_INVALID, "p2p_allgather: bad world/rank");
    if (bytes % 16 || ((uintptr_t)local & 15)) return agx_set_error(AGX_E_INVALID, "p2p_allgather: bytes and local must be 16-byte aligned");
    if (bytes == 0) return AGX_OK;
    size_t n_vec = bytes / 16;
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    long long blocks = (long long)((n_vec + 255) / 256);
    if (blocks > 2LL * sms) blocks = 2LL * sms;  // all blocks co-resident: the last one spins on peers
    p2p_allgather_kernel<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float4*>(local), peer_bufs, peer_flags,
                                                                      world, rank, n_vec, epoch, scratch);
    return agx_check_launch("p2p_allgather_kernel");
}
