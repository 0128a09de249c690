#include <stdarg.h>
#include <stdio.h>

#include "../../include/aerial_gym_b200.h"
#include <stdlib.h>

#include "agx_common.cuh"

static thread_local char g_err[512] = "";

int agx_set_error(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

int agx_check_cuda(cudaError_t e, const char* what) {
    if (e == cudaSuccess) return AGX_OK;
    return agx_set_error(AGX_E_CUDA, "%s: %s", what, cudaGetErrorString(e));
}

int agx_check_launch(const char* what) { return agx_check_cuda(cudaPeekAtLastError(), what); }

// The chained HP1 step and the gather kernels that run beside it must agree on the SM's shared-memory carve-out (see agx_common.cuh).
int agx_coresident_carveout_pct() {
    static int pct = -2;
    if (pct == -2) {
        const char* e = getenv("AGX_CARVEOUT_PCT");  // A/B knob: percent of the unified L1 / shared memory, -1 = leave the driver's choice
        pct = e ? atoi(e) : 25;
    }
    return pct;
}

extern "C" {
int agx_abi_version(void) { return AGX_ABI_VERSION; }
const char* agx_last_error(void) { return g_err; }
int agx_host_alloc(uint64_t bytes, void** out) {
    if (!out) return agx_set_error(AGX_E_NULL, "out is NULL");
    *out = nullptr;
    if (bytes == 0) return AGX_OK;
    return agx_check_cuda(cudaHostAlloc(out, (size_t)bytes, cudaHostAllocPortable | cudaHostAllocMapped), "cudaHostAlloc");
}
int agx_host_free(void* p) {
    if (!p) return AGX_OK;
    return agx_check_cuda(cudaFreeHost(p), "cudaFreeHost");
}
uint64_t agx_sizeof(int which) {
    switch (which) {
        case 0: return sizeof(AgxHp1Config);
        case 1: return sizeof(AgxHp1Buffers);
        case 2: return sizeof(AgxHp1ResetDraws);
        case 5: return sizeof(AgxNavRewardParams);
        case 6: return sizeof(AgxImuConfig);
        case 7: return sizeof(AgxLidarNavRewardParams);
        case 9: return sizeof(AgxE2ERewardParams);
        case 10: return sizeof(AgxObsGatherPush);
        case 15: return sizeof(AgxArticulation);
        case 17: return sizeof(AgxJointEffort);
#ifdef AGX_HAVE_HP2
        case 3: return sizeof(AgxHp2Scene);
        case 4: return sizeof(AgxHp2Sensor);
        case 8: return sizeof(AgxHp2Noise);
        case 11: return sizeof(AgxContactParams);
        case 12: return sizeof(AgxContactMotion);
        case 13: return sizeof(AgxObstacleMass);
        case 14: return sizeof(AgxObstacleHull);
        case 16: return sizeof(AgxObstacleBoxes);
#endif
        default: return 0;
    }
}
}
