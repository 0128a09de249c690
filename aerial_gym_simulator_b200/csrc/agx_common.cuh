// Error plumbing shared by the translation units of libaerial_gym_b200.so.
#pragma once
#include <cuda_runtime.h>

// records a thread-local message, returns `code`
int agx_set_error(int code, const char* fmt, ...);
// cudaPeekAtLastError after a launch -> AGX_OK or AGX_E_CUDA (message recorded)
int agx_check_launch(const char* what);
int agx_check_cuda(cudaError_t e, const char* what);

// Shared-memory carve-out (percent) requested by every kernel that must be CO-RESIDENT with the chained HP1 step: the step itself
// (eight 64-thread CTAs of 3.3 KB static + 1 KB reserved shared memory per SM) and the observation gather's push / gate / wait
// kernels.  Kernels on one SM share one carve-out; a push CTA that reached an idle SM first used to pin it to a small one where ~1
// step CTA fits (24 push CTAs cost > 160 CTA slots and starved the step that needs its whole grid resident).  25 % of the
// 228 KB = the 64 KB configuration: room for the eight step CTAs.
int agx_coresident_carveout_pct();
template <class K>
inline void agx_set_coresident_carveout(K kernel) {
    const int pct = agx_coresident_carveout_pct();
    if (pct >= 0) cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, pct);
}
