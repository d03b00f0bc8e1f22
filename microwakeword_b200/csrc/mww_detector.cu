// mww_detector.cu -- the streaming detector's kernels with one cutoff for every row: the update kernel's two forms
// (mww_detector.cuh) and the reset kernel.  The per-row instantiations live in mww_detector_cutoffs.cu, a library of their
// own, so that this one keeps exactly these three kernels.
#include "mww_detector.cuh"

namespace mww {

// fresh state for rows[0, n) (indices out of range ignored) or, rows == nullptr, for every row
__global__ void __launch_bounds__(kThreads) detector_reset_kernel(DetectorArgs a, const int32_t *__restrict__ rows, int n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const long long row = rows ? rows[i] : i;
    if (row < 0 || row >= a.n_rows) return;
    for (int j = 0; j < a.rule.window - 1; ++j) a.hist[(long long)j * a.n_rows + row] = 0.f;
    a.seen[row] = 0;
    a.cooldown[row] = a.rule.cooldown_slices;
}

cudaError_t launch_detector_update(const DetectorArgs &a, const float *probs, int n_steps, long long pitch, cudaStream_t st) {
    return launch_update_form<false>(a, nullptr, probs, n_steps, pitch, st);
}

cudaError_t launch_detector_reset(const DetectorArgs &a, const int32_t *rows, int n, cudaStream_t st) {
    if (n <= 0) return cudaSuccess;
    detector_reset_kernel<<<(unsigned)((n + kThreads - 1) / kThreads), kThreads, 0, st>>>(a, rows, n);
    return cudaGetLastError();
}

}  // namespace mww
