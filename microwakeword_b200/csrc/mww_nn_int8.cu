// mww_nn_int8.cu -- sm_90a kernel + launcher for the int8-quantised streaming MixedNet
// (phase functions and reference citations: mww_nn_i8_dev.cuh).
#include <cuda_runtime.h>

#include <algorithm>

#include "mww_kernels.h"

namespace mww {

__global__ void __launch_bounds__(kNnThreads, 2)
nn_i8_clip_kernel(NnWeightsI8 W, int8_t *__restrict__ state, int8_t *__restrict__ pend, int n_pend,
                  const void *__restrict__ rows, long long rows_stream_stride_bytes, int n_rows, int row_type,
                  float *__restrict__ probs, long long probs_stream_stride) {
    extern __shared__ __align__(16) int32_t smi[];
    const int tid = threadIdx.x;
    const long long s = blockIdx.x;
    int8_t *my_state = state + s * kStateFloats;
    int8_t *my_pend = pend + s * 2 * kNumChannels;
    NnInputI8 in;
    in.ring0 = my_state; in.pend = my_pend; in.n_pend = n_pend;
    in.rows = static_cast<const char *>(rows) + s * rows_stream_stride_bytes;
    in.n_rows = n_rows; in.row_type = row_type;
    const int n_virtual = n_pend + n_rows;
    const int n_steps = n_virtual / 3;

    nnq_load_state(tid, smi, my_state, W);
    nnq_load_weights(tid, smi, W);
    __syncthreads();
    for (int step0 = 0; step0 < n_steps; step0 += kTT) {
        const int n = min(kTT, n_steps - step0);
        nnq_load_features(tid, smi, in, W, step0, n);
        __syncthreads();
        nnq_first_conv_mma(tid, smi, W, n);
        __syncthreads();
        nnq_depthwise<0>(tid, smi, W); __syncthreads();
        nnq_pointwise_mma<0>(tid, smi, W, n); __syncthreads();
        nnq_depthwise<1>(tid, smi, W); __syncthreads();
        nnq_pointwise_mma<1>(tid, smi, W, n); __syncthreads();
        nnq_depthwise<2>(tid, smi, W); __syncthreads();
        nnq_pointwise_mma<2>(tid, smi, W, n); __syncthreads();
        nnq_depthwise<3>(tid, smi, W); __syncthreads();
        nnq_pointwise_mma<3>(tid, smi, W, n); __syncthreads();
        nnq_head_partial(tid, smi, W);
        __syncthreads();
        nnq_head_finish(tid, smi, W, n, probs + s * probs_stream_stride + step0);
        float tmp[5][kShiftPerThread];   // bit-copy of the int32 words
        nn_shift_read(tid, reinterpret_cast<const float *>(smi), n, tmp);
        __syncthreads();
        nn_shift_write(tid, reinterpret_cast<float *>(smi), tmp);
        __syncthreads();
    }
    NnTailI8 tail;
    nnq_tail_read(tid, in, W, n_steps, n_virtual, tail);
    __syncthreads();
    nnq_tail_write(tid, smi, my_state, my_pend, W, tail);
}

// ids == nullptr: streams 0 .. n; otherwise the n listed streams (ids outside [0, n_streams) are skipped)
__global__ void fill_state_i8_kernel(NnWeightsI8 W, int8_t *__restrict__ state, int8_t *__restrict__ pend, const int32_t *__restrict__ ids, int n,
                                     int n_streams) {
    const long long total = (long long)n * (kStateFloats + 2 * kNumChannels);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long k = i / (kStateFloats + 2 * kNumChannels);
        const int e = (int)(i - k * (kStateFloats + 2 * kNumChannels));
        const long long s = ids ? ids[k] : k;
        if (s < 0 || s >= n_streams) continue;
        if (e < kStateFloats) state[s * kStateFloats + e] = nnq_reset_value(W, e);
        else pend[s * 2 * kNumChannels + (e - kStateFloats)] = (int8_t)W.zp[0];
    }
}

cudaError_t launch_nn_i8(const NnWeightsI8 &W, int8_t *state, int8_t *pend, int n_pend, const void *rows,
                         long long rows_stream_stride_bytes, int n_rows, int row_type, float *probs,
                         long long probs_stream_stride, int n_streams, cudaStream_t st) {
    if (n_streams <= 0) return cudaSuccess;
    static bool attr_done[64] = {};
    if (first_launch_on_this_device(attr_done)) {
        cudaError_t e = cudaFuncSetAttribute(nn_i8_clip_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kNnI8SmemBytes);
        if (e != cudaSuccess) return e;
    }
    nn_i8_clip_kernel<<<(unsigned)n_streams, kNnThreads, kNnI8SmemBytes, st>>>(W, state, pend, n_pend, rows, rows_stream_stride_bytes, n_rows,
                                                                            row_type, probs, probs_stream_stride);
    return cudaGetLastError();
}

cudaError_t launch_fill_state_i8(const NnWeightsI8 &W, int8_t *state, int8_t *pend, const int32_t *ids, int n, int n_streams, cudaStream_t st) {
    if (n <= 0) return cudaSuccess;
    const long long total = (long long)n * (kStateFloats + 2 * kNumChannels);
    const unsigned blocks = (unsigned)std::min<long long>((total + 255) / 256, 132 * 16);
    fill_state_i8_kernel<<<blocks, 256, 0, st>>>(W, state, pend, ids, n, n_streams);
    return cudaGetLastError();
}

}  // namespace mww
