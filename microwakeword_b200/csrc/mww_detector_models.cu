// mww_detector_models.cu -- the multi-model streaming detector's kernels in uniform mode: the update kernel over plain
// descriptors (mww_detector_models.cuh) and the reset kernel.  The per-row instantiation lives in mww_detector_cutoffs.cu,
// a library of its own, so that this one keeps exactly these two kernels.
// detector_models_reset_kernel: a thread per listed stream resets that stream's row of every model.
#include "mww_detector_models.cuh"

namespace mww {

// fresh state for the streams ids[0, n) (out of range ignored) or, ids == nullptr, for streams [0, n)
__global__ void __launch_bounds__(kModelsThreads) detector_models_reset_kernel(const __grid_constant__ DetectModelsArgs a,
                                                                               const int32_t *__restrict__ ids, int n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    detect_models_reset_stream(a, ids ? ids[i] : i);
}

cudaError_t launch_detector_models_update(const DetectModelsArgs &a, cudaStream_t st) { return launch_models_update_form(a, st); }

cudaError_t launch_detector_models_reset(const DetectModelsArgs &a, const int32_t *ids, int n, cudaStream_t st) {
    if (n <= 0) return cudaSuccess;
    detector_models_reset_kernel<<<(unsigned)((n + kModelsThreads - 1) / kModelsThreads), kModelsThreads, 0, st>>>(a, ids, n);
    return cudaGetLastError();
}

}  // namespace mww
