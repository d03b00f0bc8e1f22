// mww_detect.cu -- detection post-processing on the GPU (SURVEY.md 8 f-1): what the reference's evaluation
// harness does with the per-step probabilities right after Model.predict_spectrogram
//   moving average ............ microwakeword/test.py:337-341  (sliding_window_view(p, L).mean(-1), L = 5)
//   false-accept counting ..... microwakeword/test.py:118-135  (per cutoff: cooldown, re-armed by a detection)
//   positive-sample score ..... microwakeword/test.py:364-373  (max of the moving average after the first
//                               `ignore_slices_after_accept` probabilities)
//   accuracy counts ........... microwakeword/test.py:452-484  (tflite_model_accuracy: 0.5 crossings per ambient track,
//                               last probability > 0.5 per test clip)
// Keeping this on the device means only detections / scores leave the GPU instead of every probability.
// Parity is PINNED: tests/golden/detection_golden.npz comes from executing the reference's own function.
#include <cuda_runtime.h>
#include <math.h>

#include <algorithm>

#include "../../include/mww.h"

namespace {

// float32 sequential sum then one IEEE division, exactly NumPy's float32 mean over a length-L axis
__device__ __forceinline__ float window_mean(const float *p, int window) {
    float s = p[0];
    for (int j = 1; j < window; ++j) s = __fadd_rn(s, p[j]);
    return __fdiv_rn(s, (float)window);
}

// one thread per (track, output position): tracks on grid x (up to 2^31 - 1 of them), positions on grid y and a grid stride
__global__ void moving_average_kernel(const float *__restrict__ probs, const long long *__restrict__ offsets,
                                      const int *__restrict__ lengths, int n_tracks, int window, float *__restrict__ out,
                                      const long long *__restrict__ out_offsets) {
    const int trk = blockIdx.x;
    if (trk >= n_tracks) return;
    const int n = lengths[trk] - window + 1;
    const float *p = probs + offsets[trk];
    float *o = out + out_offsets[trk];
    for (int i = blockIdx.y * blockDim.x + threadIdx.x; i < n; i += gridDim.y * blockDim.x) o[i] = window_mean(p + i, window);
}

// one thread per (track, cutoff): the cooldown chain is sequential in time (test.py:120-135)
__global__ void false_accept_kernel(const float *__restrict__ probs, const long long *__restrict__ offsets,
                                    const int *__restrict__ lengths, int n_tracks, int window, const double *__restrict__ cutoffs,
                                    int n_cutoffs, int ignore, int *__restrict__ counts) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)n_tracks * n_cutoffs) return;
    const int trk = (int)(idx / n_cutoffs), ci = (int)(idx - (long long)trk * n_cutoffs);
    const double cutoff = cutoffs[ci];
    const int n = lengths[trk] - window + 1;
    const float *p = probs + offsets[trk];
    int cooldown = ignore, count = 0;
    for (int i = 0; i < n; ++i) {
        cooldown = cooldown > 0 ? cooldown - 1 : 0;
        const double v = (double)window_mean(p + i, window);   // float32 probability compared against a float64 cutoff
        if (cooldown == 0 && v > cutoff) { ++count; cooldown = ignore; }
    }
    counts[idx] = count;
}

// one warp per track: max of the moving average over probs[ignore:], NaN when fewer than `window` remain
__global__ void positive_score_kernel(const float *__restrict__ probs, const long long *__restrict__ offsets,
                                      const int *__restrict__ lengths, int n_tracks, int window, int ignore, float *__restrict__ score) {
    const int trk = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
    if (trk >= n_tracks) return;
    const int lane = threadIdx.x & 31;
    const int n = lengths[trk] - ignore - window + 1;
    const float *p = probs + offsets[trk] + ignore;
    float m = -INFINITY;
    for (int i = lane; i < n; i += 32) m = fmaxf(m, window_mean(p + i, window));
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (lane == 0) score[trk] = n > 0 ? m : NAN;
}

// one warp per track, 32 consecutive steps per pass (coalesced): whether step i is a rising crossing prev <= 0.5 < p
// (test.py:479) does not depend on the chain, so the lanes find the crossings in parallel and only the min_gap chain over
// the crossings (last_positive_index, :480-483) is walked in order -- by every lane alike, from the same ballot mask.
__global__ void accuracy_kernel(const float *__restrict__ probs, const long long *__restrict__ offsets, const int *__restrict__ lengths,
                                int n_tracks, int min_gap, int *__restrict__ false_accepts, int *__restrict__ last_positive) {
    const int trk = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
    if (trk >= n_tracks) return;
    const int lane = threadIdx.x & 31;
    const int n = lengths[trk];
    const float *p = probs + offsets[trk];
    if (false_accepts) {
        int last = 0, count = 0;                                // previous_probability and last_positive_index restart at 0 (:475-476)
        for (int base = 0; base < n; base += 32) {
            const int i = base + lane;
            const bool crossing = i < n && (i == 0 ? 0.f : p[i - 1]) <= 0.5f && p[i] > 0.5f;
            for (unsigned mask = __ballot_sync(0xffffffffu, crossing); mask; mask &= mask - 1) {
                const int j = base + __ffs(mask) - 1;
                if (j - last > min_gap) { ++count; last = j; }
            }
        }
        if (lane == 0) false_accepts[trk] = count;
    }
    if (last_positive && lane == 0) last_positive[trk] = (n > 0 && p[n - 1] > 0.5f) ? 1 : 0;   // probabilities[-1] > 0.5 (:462-463)
}

}  // namespace

extern "C" {

int mww_moving_average(const float *d_probs, const long long *d_offsets, const int *d_lengths, int n_tracks, int max_length, int window,
                       float *d_out, const long long *d_out_offsets, void *cu_stream) {
    if (!d_probs || !d_offsets || !d_lengths || !d_out || !d_out_offsets || window < 1 || n_tracks < 0) return MWW_EINVAL;
    if (n_tracks == 0) return MWW_OK;
    // grid y is capped at 65 535 by CUDA: longer tracks are covered by the kernel's grid stride
    const long long chunks = std::min(std::max(((long long)max_length + 255) / 256, 1ll), 65535ll);
    dim3 grid((unsigned)n_tracks, (unsigned)chunks);
    moving_average_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(cu_stream)>>>(d_probs, d_offsets, d_lengths, n_tracks, window, d_out, d_out_offsets);
    return cudaGetLastError() == cudaSuccess ? MWW_OK : MWW_ECUDA;
}

int mww_false_accept_counts(const float *d_probs, const long long *d_offsets, const int *d_lengths, int n_tracks, int window,
                            const double *d_cutoffs, int n_cutoffs, int ignore_slices_after_accept, int *d_counts, void *cu_stream) {
    if (!d_probs || !d_offsets || !d_lengths || !d_cutoffs || !d_counts || window < 1 || n_tracks < 0 || n_cutoffs < 1) return MWW_EINVAL;
    if (n_tracks == 0) return MWW_OK;
    const long long total = (long long)n_tracks * n_cutoffs;
    false_accept_kernel<<<(unsigned)((total + 127) / 128), 128, 0, static_cast<cudaStream_t>(cu_stream)>>>(
        d_probs, d_offsets, d_lengths, n_tracks, window, d_cutoffs, n_cutoffs, ignore_slices_after_accept, d_counts);
    return cudaGetLastError() == cudaSuccess ? MWW_OK : MWW_ECUDA;
}

int mww_positive_scores(const float *d_probs, const long long *d_offsets, const int *d_lengths, int n_tracks, int window,
                        int ignore_slices_after_accept, float *d_scores, void *cu_stream) {
    if (!d_probs || !d_offsets || !d_lengths || !d_scores || window < 1 || n_tracks < 0) return MWW_EINVAL;
    if (n_tracks == 0) return MWW_OK;
    positive_score_kernel<<<(unsigned)((n_tracks + 3) / 4), 128, 0, static_cast<cudaStream_t>(cu_stream)>>>(
        d_probs, d_offsets, d_lengths, n_tracks, window, ignore_slices_after_accept, d_scores);
    return cudaGetLastError() == cudaSuccess ? MWW_OK : MWW_ECUDA;
}

int mww_accuracy_counts(const float *d_probs, const long long *d_offsets, const int *d_lengths, int n_tracks, int min_gap,
                        int *d_false_accepts, int *d_last_positive, void *cu_stream) {
    if (!d_probs || !d_offsets || !d_lengths || n_tracks < 0) return MWW_EINVAL;
    if (n_tracks == 0 || (!d_false_accepts && !d_last_positive)) return MWW_OK;
    accuracy_kernel<<<(unsigned)((n_tracks + 3) / 4), 128, 0, static_cast<cudaStream_t>(cu_stream)>>>(
        d_probs, d_offsets, d_lengths, n_tracks, min_gap, d_false_accepts, d_last_positive);
    return cudaGetLastError() == cudaSuccess ? MWW_OK : MWW_ECUDA;
}

}  // extern "C"
