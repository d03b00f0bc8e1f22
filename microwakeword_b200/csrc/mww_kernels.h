// mww_kernels.h -- launcher prototypes shared by the C-ABI layer (mww_capi.cu) and the kernel files.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "mww_tables.h"

namespace mww {

// Dynamic shared memory above 48 KB is opt-in per kernel AND per device (cudaFuncSetAttribute applies to the current
// device only): a process that drives several GPUs must opt in on each of them.  `done` is the launcher's static flag set.
inline bool first_launch_on_this_device(bool (&done)[64]) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return true;
    if (done[dev]) return false;
    done[dev] = true;
    return true;
}

// Every launcher that reads caller audio is instantiated for T = int16_t (PCM) and T = float (float32 in [-1, 1], converted
// on load with pcm16_from_f32); the window carry is int16 either way, so calls of both types can follow each other.
template <typename T>
cudaError_t launch_k1(const FrontendParams &P, const int16_t *carry, int used, const T *audio,
                      long long audio_stride, int n_samples, int n_streams, int n_frames, uint32_t *vout, int sm_count,
                      cudaStream_t st);
// long calls with enough streams for one CTA per stream: K1 + the temporal chain in one launch, features written directly
// (no V scratch).  frontend_clip_fuses() is the predicate the C-ABI layer sizes its scratch with.
bool frontend_clip_fuses(int n_streams, int n_frames, int sm_count);
template <typename T>
cudaError_t launch_frontend_clip_fused(const FrontendParams &P, const int16_t *carry, int used, const T *audio, long long audio_stride,
                                       int n_samples, int n_streams, int n_frames, uint32_t *estimate, uint16_t *feat, long long feat_stream_stride,
                                       cudaStream_t st);
// any even hop <= 480 samples (window_step != 10 ms): K1 + temporal chain, one CTA per stream, features written directly
template <typename T>
cudaError_t launch_frontend_hop(const FrontendParams &P, const int16_t *carry, int used, const T *audio, long long audio_stride,
                                int n_samples, int n_streams, int n_frames, int hop, uint32_t *estimate, uint16_t *feat,
                                long long feat_stream_stride, cudaStream_t st);
// short calls (<= 8 frames per stream, <= 2 hops left over): K1 + K2 + carry update in one launch
bool frontend_fusable(int used, int n_samples, int n_frames);
template <typename T>
cudaError_t launch_frontend_fused(const FrontendParams &P, int16_t *carry, int used, const T *audio,
                                  long long audio_stride, int n_samples, int n_streams, int n_frames, uint32_t *estimate, uint16_t *feat,
                                  long long feat_stream_stride, cudaStream_t st);
cudaError_t launch_k2(const FrontendParams &P, const uint32_t *vin, int n_streams, int n_frames, uint32_t *estimate,
                      uint16_t *feat, long long feat_stream_stride, cudaStream_t st);
template <typename T>
cudaError_t launch_carry_update(int16_t *carry, int used, const T *audio, long long audio_stride, int n_samples,
                                int n_streams, int consumed, int new_used, cudaStream_t st);

}  // namespace mww

#include "mww_nn_dev.cuh"
namespace mww {
cudaError_t launch_nn_f32(const NnWeightsF32 &W, float *state, float *pend, int n_pend, const void *rows,
                          long long rows_stream_stride_bytes, int n_rows, int rows_are_f32, float *probs,
                          long long probs_stream_stride, float *logits, int n_streams, cudaStream_t st);
}  // namespace mww

#include "mww_nn_i8_dev.cuh"
namespace mww {
cudaError_t launch_nn_i8(const NnWeightsI8 &W, int8_t *state, int8_t *pend, int n_pend, const void *rows,
                         long long rows_stream_stride_bytes, int n_rows, int row_type, float *probs,
                         long long probs_stream_stride, int n_streams, cudaStream_t st);
// zero-point fill of streams 0 .. n (ids == nullptr) or of the n listed streams
cudaError_t launch_fill_state_i8(const NnWeightsI8 &W, int8_t *state, int8_t *pend, const int32_t *ids, int n, int n_streams, cudaStream_t st);
}  // namespace mww

#include "mww_nn_live.cuh"
namespace mww {
// live-step path (one model step for many streams per launch; mww_nn_live.cuh).  `heads` = current rotation of the rings;
// the caller advances every head by one (mod its ring length) after the launch.
cudaError_t launch_nn_f32_live(const NnWeightsF32 &W, float *state, float *pend, int n_pend, const void *rows,
                               long long rows_stream_stride_bytes, int rows_are_f32, float *probs, long long probs_stride,
                               int n_streams, const LiveHeads &heads, int sm_count, int variant, cudaStream_t st);
// rotate every ring of every stream back to the canonical oldest-first layout (no-op rings with head 0 are skipped)
cudaError_t launch_nn_live_canonicalise(float *state, int n_streams, const LiveHeads &heads, cudaStream_t st);
// int8 live-step path (mww_nn_i8_live.cuh); rows must be 16-byte aligned with a 16-byte-multiple stream stride
cudaError_t launch_nn_i8_live(const NnWeightsI8 &W, int8_t *state, int8_t *pend, int n_pend, const void *rows,
                              long long rows_stream_stride_bytes, int row_type, float *probs, long long probs_stride, int n_streams,
                              const LiveHeads &heads, int sm_count, cudaStream_t st);
cudaError_t launch_nn_i8_live_canonicalise(int8_t *state, int n_streams, const LiveHeads &heads, cudaStream_t st);
}  // namespace mww

#include "mww_nn_generic.cuh"
namespace mww {
// run-time-geometry MixedNet (any architecture other than the compiled-in okay_nabu one; mww_nn_generic.cuh)
cudaError_t launch_nn_generic_f32(const GenArch &A, const GenWeightsF32 &W, float *state, float *pend, int n_pend, const void *rows,
                                  long long rows_stream_stride_bytes, int n_rows, int row_type, float *probs, long long probs_stream_stride,
                                  int n_streams, cudaStream_t st);
cudaError_t launch_nn_generic_i8(const GenArch &A, const GenWeightsI8 &W, int8_t *state, int8_t *pend, int n_pend, const void *rows,
                                 long long rows_stream_stride_bytes, int n_rows, int row_type, float *probs, long long probs_stream_stride,
                                 int n_streams, cudaStream_t st);
cudaError_t launch_gen_fill_state_i8(const GenArch &A, const GenWeightsI8 &W, int8_t *state, int8_t *pend, int n, const int32_t *ids, int n_streams,
                                     cudaStream_t st);
}  // namespace mww
