// agx_hp2_noise_limits: the ray-cast sensors' noise model + range limits + normalisation as one in-place pass with a
// counter-based device RNG (noise_core.cuh).  HBM-bound: 4 B read + 4 B written per value (the reference's torch version
// moves ~10x that).  One thread per pixel, grid-stride so any image size fits one launch.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/aerial_gym_b200.h"
#include "agx_common.cuh"
#include "noise_core.cuh"

namespace {
using namespace agx;
constexpr int kNoiseThreads = 256;

__global__ void __launch_bounds__(kNoiseThreads)
noise_limits_kernel(float* __restrict__ pixels, uint64_t num_pixels, uint64_t first_pixel, const __grid_constant__ AgxHp2Noise n, uint32_t frame, uint32_t k0,
                    uint32_t k1) {
    const uint64_t step = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < num_pixels; i += step)
        noise_limits_pixel(i, first_pixel + i, pixels, n, frame, k0, k1);
}
}  // namespace

extern "C" int agx_hp2_noise_limits(float* pixels, uint64_t num_pixels, uint64_t first_pixel, const AgxHp2Noise* cfg, uint64_t seed,
                                    uint32_t frame, void* stream) {
    if (!cfg) return agx_set_error(AGX_E_NULL, "agx_hp2_noise_limits: cfg is NULL");
    if (cfg->components != 1 && cfg->components != 3) return agx_set_error(AGX_E_INVALID, "agx_hp2_noise_limits: components must be 1 or 3");
    if (cfg->normalize && !(cfg->max_range > 0.0f)) return agx_set_error(AGX_E_INVALID, "agx_hp2_noise_limits: max_range must be > 0");
    if (num_pixels == 0) return AGX_OK;
    if (!pixels) return agx_set_error(AGX_E_NULL, "agx_hp2_noise_limits: pixels is NULL");
    const uint64_t want = (num_pixels + kNoiseThreads - 1) / kNoiseThreads;
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const uint64_t cap = (uint64_t)sms * 32;  // <= 32 CTAs per SM worth of grid-stride work
    const int blocks = (int)(want < cap ? want : cap);
    noise_limits_kernel<<<blocks, kNoiseThreads, 0, (cudaStream_t)stream>>>(pixels, num_pixels, first_pixel, *cfg, frame, (uint32_t)(seed & 0xffffffffu),
                                                                           (uint32_t)(seed >> 32));
    return agx_check_launch("noise_limits_kernel");
}
