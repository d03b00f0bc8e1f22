// mww_nn_i8_live.cu -- sm_90a kernel + launcher of the int8 live-step MixedNet (phase functions and rationale:
// mww_nn_i8_live.cuh).
#include <cuda_runtime.h>

#include <algorithm>

#include "mww_kernels.h"
#include "mww_nn_i8_live.cuh"

namespace mww {

// persistent CTAs: each walks groups of 32 streams; all IMMA weights are staged once per CTA
__global__ void __launch_bounds__(kLiveQThreads, 4)
nn_i8_live_kernel(NnWeightsI8 W, int8_t *__restrict__ state, int8_t *__restrict__ pend, int n_pend, const void *__restrict__ rows,
                  long long rows_stream_stride_bytes, int row_type, float *__restrict__ probs, long long probs_stride, int n_streams,
                  LiveHeads heads) {
    extern __shared__ __align__(16) uint8_t smb[];
    const int tid = threadIdx.x;
    LiveInputI8 in;
    in.state = state; in.pend = pend; in.n_pend = n_pend; in.rows = rows;
    in.rows_stream_stride_bytes = rows_stream_stride_bytes; in.row_type = row_type;
    livq_load_weights(tid, smb, W);
    __syncthreads();
    const int n_groups = (n_streams + kLiveStreams - 1) / kLiveStreams;
    for (int g = blockIdx.x; g < n_groups; g += gridDim.x) {
        const long long s0 = (long long)g * kLiveStreams;
        const int n_valid = min(kLiveStreams, n_streams - (int)s0);
        uint32_t keep[4][kLqKeep];
        livq_build_a(tid, smb, in, W, s0, n_valid, keep);
        __syncthreads();
        livq_write_tail(tid, state, pend, s0, n_valid, keep);
        livq_first_conv_mma(tid, smb, W);
        __syncthreads();
        livq_depthwise<0>(tid, smb, W, state, s0, n_valid, heads.h[0]); __syncthreads();
        livq_pointwise_mma<0>(tid, smb, W); __syncthreads();
        livq_depthwise<1>(tid, smb, W, state, s0, n_valid, heads.h[1]); __syncthreads();
        livq_pointwise_mma<1>(tid, smb, W); __syncthreads();
        livq_depthwise<2>(tid, smb, W, state, s0, n_valid, heads.h[2]); __syncthreads();
        livq_pointwise_mma<2>(tid, smb, W); __syncthreads();
        livq_depthwise<3>(tid, smb, W, state, s0, n_valid, heads.h[3]); __syncthreads();
        livq_pointwise_mma<3>(tid, smb, W); __syncthreads();
        livq_head_partial(tid, smb, W, state, s0, n_valid, heads.h[4]);
        __syncthreads();
        livq_head_finish(tid, smb, W, s0, n_valid, probs, probs_stride);
        __syncthreads();                   // the head's partial sums live in the window buffer the next group overwrites
    }
}

cudaError_t launch_nn_i8_live(const NnWeightsI8 &W, int8_t *state, int8_t *pend, int n_pend, const void *rows,
                              long long rows_stream_stride_bytes, int row_type, float *probs, long long probs_stride, int n_streams,
                              const LiveHeads &heads, int sm_count, cudaStream_t st) {
    if (n_streams <= 0) return cudaSuccess;
    const int n_groups = (n_streams + kLiveStreams - 1) / kLiveStreams;
    const int grid = std::min(n_groups, 4 * sm_count);
    nn_i8_live_kernel<<<grid, kLiveQThreads, kLiveQSmemBytes, st>>>(W, state, pend, n_pend, rows, rows_stream_stride_bytes, row_type, probs,
                                                                   probs_stride, n_streams, heads);
    return cudaGetLastError();
}

__global__ void nn_i8_live_canonicalise_kernel(int8_t *__restrict__ state, int n_streams, LiveHeads heads) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (long long)n_streams * 288) return;
    livq_canonicalise_column(state, e / 288, (int)(e % 288), heads);
}

cudaError_t launch_nn_i8_live_canonicalise(int8_t *state, int n_streams, const LiveHeads &heads, cudaStream_t st) {
    if (n_streams <= 0) return cudaSuccess;
    const long long total = (long long)n_streams * 288;
    nn_i8_live_canonicalise_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(state, n_streams, heads);
    return cudaGetLastError();
}

}  // namespace mww
