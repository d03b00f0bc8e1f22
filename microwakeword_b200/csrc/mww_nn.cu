// mww_nn.cu -- sm_90a kernel + launcher for the fp32 streaming MixedNet in clip formulation
// (phase functions and reference citations: mww_nn_dev.cuh).
#include <cuda_runtime.h>
#include <cstdlib>

#include "mww_kernels.h"
#include "mww_nn_mma.cuh"

namespace mww {

// grid = streams; one CTA (128 threads) owns one stream for the whole call, ring state stays in
// shared memory across chunks of kTT steps.
__global__ void __launch_bounds__(kNnThreads, 2)
nn_f32_clip_kernel(NnWeightsF32 W, float *__restrict__ state, float *__restrict__ pend, int n_pend,
                   const void *__restrict__ rows, long long rows_stream_stride_bytes, int n_rows, int rows_are_f32,
                   float *__restrict__ probs, long long probs_stream_stride, float *__restrict__ logits) {
    extern __shared__ __align__(16) float sm[];
    const int tid = threadIdx.x;
    const long long s = blockIdx.x;
    float *my_state = state + s * kStateFloats;
    float *my_pend = pend + s * 2 * kNumChannels;
    NnInput in;
    in.ring0 = my_state;
    in.pend = my_pend;
    in.n_pend = n_pend;
    in.rows = static_cast<const char *>(rows) + s * rows_stream_stride_bytes;
    in.n_rows = n_rows;
    in.rows_are_f32 = rows_are_f32;
    const int n_virtual = n_pend + n_rows;
    const int n_steps = n_virtual / 3;

    nn_load_state(tid, sm, my_state);                 // cp.async group 0: lands while the first chunk's features load
    nn_commit_group();
    for (int step0 = 0; step0 < n_steps; step0 += kTT) {
        const int n = min(kTT, n_steps - step0);
        nn_load_features(tid, sm, in, step0, n);
        __syncthreads();
        float fc[4][4];
        nn_first_conv_mma_a(tid, sm, W, fc, n);
        __syncthreads();
        nn_first_conv_mma_b(tid, sm, fc, n);
        nn_stage_pw_weights<0>(tid, sm, W);          // feature planes are dead: block 0's weights land there
        nn_stage_pw_weights<1>(tid, sm, W);
        nn_wait_weights<2>();                         // first chunk: the ring-state group is complete (only the two weight groups may be in flight)
        __syncthreads();
        nn_depthwise<0>(tid, sm, W); nn_wait_weights<1>(); __syncthreads();
        nn_pointwise_mma<0>(tid, sm, W, n); __syncthreads();
        nn_stage_pw_weights<2>(tid, sm, W);          // buffer of block 0 is free again
        nn_depthwise<1>(tid, sm, W); nn_wait_weights<1>(); __syncthreads();
        nn_pointwise_mma<1>(tid, sm, W, n); __syncthreads();
        nn_stage_pw_weights<3>(tid, sm, W);
        nn_depthwise<2>(tid, sm, W); nn_wait_weights<1>(); __syncthreads();
        nn_pointwise_mma<2>(tid, sm, W, n); __syncthreads();
        nn_depthwise<3>(tid, sm, W); nn_wait_weights<0>(); __syncthreads();
        nn_pointwise_mma<3>(tid, sm, W, n); __syncthreads();
        nn_head_partial(tid, sm, W);
        __syncthreads();
        nn_head_finish(tid, sm, W, n, probs + s * probs_stream_stride + step0,
                       logits ? logits + s * probs_stream_stride + step0 : nullptr);
        float tmp[5][kShiftPerThread];
        nn_shift_read(tid, sm, n, tmp);
        __syncthreads();
        nn_shift_write(tid, sm, tmp);
        __syncthreads();
    }
    NnTail tail;
    nn_tail_read(tid, in, n_steps, n_virtual, tail);
    nn_wait_weights<0>();                             // a call without a full step still has the ring-state copy in flight
    __syncthreads();
    nn_tail_write(tid, sm, my_state, my_pend, tail);
}

cudaError_t launch_nn_f32(const NnWeightsF32 &W, float *state, float *pend, int n_pend, const void *rows,
                          long long rows_stream_stride_bytes, int n_rows, int rows_are_f32, float *probs,
                          long long probs_stream_stride, float *logits, int n_streams, cudaStream_t st) {
    if (n_streams <= 0) return cudaSuccess;
    static bool attr_done[64] = {};
    static int pad = 0;
    if (first_launch_on_this_device(attr_done)) {
        if (const char *e = getenv("MWW_NN_SMEM_PAD")) pad = atoi(e);       // experiment: force 1 CTA / SM
        cudaError_t e = cudaFuncSetAttribute(nn_f32_clip_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kNnSmemBytes + pad);
        if (e != cudaSuccess) return e;
    }
    nn_f32_clip_kernel<<<(unsigned)n_streams, kNnThreads, kNnSmemBytes + pad, st>>>(W, state, pend, n_pend, rows, rows_stream_stride_bytes,
                                                                             n_rows, rows_are_f32, probs, probs_stream_stride, logits);
    return cudaGetLastError();
}

}  // namespace mww
