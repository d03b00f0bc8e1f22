// mww_nn_generic.cu -- sm_90a kernels + launchers of the run-time-geometry MixedNet (phase functions, rationale and
// reference citations: mww_nn_generic.cuh).  One CTA = one stream, stepped like the reference's interpreter loop
// (microwakeword/inference.py:109-123) with every ring resident in shared memory for the whole call.
#include <cuda_runtime.h>

#include "mww_kernels.h"
#include "mww_nn_generic.cuh"

namespace mww {

namespace {
MWW_D void gen_advance(int &pos, int slots) { pos = pos + 1 == slots ? 0 : pos + 1; }
}  // namespace

__global__ void __launch_bounds__(kGenThreads)
nn_generic_f32_kernel(GenArch A, GenWeightsF32 W, float *__restrict__ state, float *__restrict__ pend, int n_pend,
                      const void *__restrict__ rows, long long rows_stream_stride_bytes, int n_rows, int row_type,
                      float *__restrict__ probs, long long probs_stream_stride) {
    extern __shared__ __align__(16) float gsm[];
    const int tid = threadIdx.x;
    const long long s = blockIdx.x;
    float *my_state = state + s * A.state_elems;
    float *my_pend = pend + s * (long long)A.pend_cap * kNumChannels;
    GenInput<float> in;
    in.state = my_state; in.pend = my_pend; in.n_pend = n_pend;
    in.rows = static_cast<const char *>(rows) + s * rows_stream_stride_bytes;
    in.n_rows = n_rows; in.row_type = row_type;
    const int n_steps = (n_pend + n_rows) / A.stride;
    int pos[kGenMaxBlocks + 1];
#pragma unroll
    for (int i = 0; i <= kGenMaxBlocks; ++i) pos[i] = 0;

    gen_f32_load_state(tid, gsm, A, my_state);
    __syncthreads();
    for (int t = 0; t < n_steps; ++t) {
        gen_f32_window(tid, gsm, A, in, t);
        __syncthreads();
        gen_f32_first_conv(tid, gsm, A, W);
        __syncthreads();
        for (int b = 0; b < A.n_blocks; ++b) {
            gen_f32_depthwise(tid, gsm, A, W, b, pos[b]);
            gen_advance(pos[b], A.kmax[b]);
            __syncthreads();
            gen_f32_pointwise(tid, gsm, A, W, b);
            __syncthreads();
        }
        gen_f32_head_partial(tid, gsm, A, W, pos[A.n_blocks]);
        gen_advance(pos[A.n_blocks], A.head_rows);
        __syncthreads();
        gen_f32_head_finish(tid, gsm, A, W, probs + s * probs_stream_stride + t);
        // the next writer of d[] (depthwise of block 0) is two barriers away from this read
    }
    gen_f32_tail_gather(tid, gsm, A, in, n_steps);
    __syncthreads();
    gen_f32_tail_store(tid, gsm, A, my_state, my_pend, A.ring0 + n_pend + n_rows - A.stride * n_steps, pos);
}

__global__ void __launch_bounds__(kGenThreads)
nn_generic_i8_kernel(GenArch A, GenWeightsI8 W, int8_t *__restrict__ state, int8_t *__restrict__ pend, int n_pend,
                     const void *__restrict__ rows, long long rows_stream_stride_bytes, int n_rows, int row_type,
                     float *__restrict__ probs, long long probs_stream_stride) {
    extern __shared__ __align__(16) int32_t gsmi[];
    const int tid = threadIdx.x;
    const long long s = blockIdx.x;
    int8_t *my_state = state + s * A.state_elems;
    int8_t *my_pend = pend + s * (long long)A.pend_cap * kNumChannels;
    GenInput<int8_t> in;
    in.state = my_state; in.pend = my_pend; in.n_pend = n_pend;
    in.rows = static_cast<const char *>(rows) + s * rows_stream_stride_bytes;
    in.n_rows = n_rows; in.row_type = row_type;
    const int n_steps = (n_pend + n_rows) / A.stride;
    int pos[kGenMaxBlocks + 1];
#pragma unroll
    for (int i = 0; i <= kGenMaxBlocks; ++i) pos[i] = 0;

    gen_i8_load_state(tid, gsmi, A, my_state);
    __syncthreads();
    for (int t = 0; t < n_steps; ++t) {
        gen_i8_window(tid, gsmi, A, W, in, t);
        __syncthreads();
        gen_i8_first_conv(tid, gsmi, A, W);
        __syncthreads();
        for (int b = 0; b < A.n_blocks; ++b) {
            gen_i8_depthwise(tid, gsmi, A, W, b, pos[b]);
            gen_advance(pos[b], A.kmax[b]);
            __syncthreads();
            gen_i8_pointwise(tid, gsmi, A, W, b);
            __syncthreads();
        }
        gen_i8_head_partial(tid, gsmi, A, W, pos[A.n_blocks]);
        gen_advance(pos[A.n_blocks], A.head_rows);
        __syncthreads();
        gen_i8_head_finish(tid, gsmi, A, W, probs + s * probs_stream_stride + t);
    }
    gen_i8_tail_gather(tid, gsmi, A, W, in, n_steps);
    __syncthreads();
    gen_i8_tail_store(tid, gsmi, A, my_state, my_pend, A.ring0 + n_pend + n_rows - A.stride * n_steps, pos);
}

// fp32 graph with hybrid (int8-weight) ops: the fp32 kernel's structure and state layout; every hybrid op adds three
// phases (min / max partials, scale + zero point, quantisation) ahead of its int32 contraction (mww_nn_generic.cuh)
__global__ void __launch_bounds__(kGenThreads)
nn_generic_hybrid_kernel(GenArch A, GenWeightsF32 W, GenHybrid H, float *__restrict__ state, float *__restrict__ pend, int n_pend,
                         const void *__restrict__ rows, long long rows_stream_stride_bytes, int n_rows, int row_type,
                         float *__restrict__ probs, long long probs_stream_stride) {
    extern __shared__ __align__(16) float gsmh[];
    const int tid = threadIdx.x;
    const long long s = blockIdx.x;
    float *my_state = state + s * A.state_elems;
    float *my_pend = pend + s * (long long)A.pend_cap * kNumChannels;
    GenInput<float> in;
    in.state = my_state; in.pend = my_pend; in.n_pend = n_pend;
    in.rows = static_cast<const char *>(rows) + s * rows_stream_stride_bytes;
    in.n_rows = n_rows; in.row_type = row_type;
    const int n_steps = (n_pend + n_rows) / A.stride;

    gen_f32_load_state(tid, gsmh, A, my_state);
    __syncthreads();
    for (int t = 0; t < n_steps; ++t) {
        if (H.mode0 != kHyFloat) {
            gen_hy_window(tid, gsmh, A, H, in, t);
            __syncthreads();
            gen_hy_qparams(tid, gsmh, H, tid == 0 ? H.mode0 : kHyFloat);
            __syncthreads();
            gen_hy_quant_window(tid, gsmh, A, H);
            __syncthreads();
            gen_hy_first_conv(tid, gsmh, A, H);
        } else {
            gen_f32_window(tid, gsmh, A, in, t);
            __syncthreads();
            gen_f32_first_conv(tid, gsmh, A, W);
        }
        __syncthreads();
        for (int b = 0; b < A.n_blocks; ++b) {
            const int pos = t % A.kmax[b];                  // ring slot of the new row: every ring starts the call at slot 0
            if (H.any_dw[b]) {
                gen_hy_block_insert(tid, gsmh, A, H, b, pos);
                __syncthreads();
                gen_hy_qparams(tid, gsmh, H, tid < H.n_groups[b] ? H.g_mode[b][tid & (kHyMaxQ - 1)] : kHyFloat);
                __syncthreads();
                gen_hy_quant_block(tid, gsmh, A, H, b, pos);
                __syncthreads();
                gen_hy_depthwise(tid, gsmh, A, W, H, b, pos);
            } else {
                gen_f32_depthwise(tid, gsmh, A, W, b, pos);
            }
            __syncthreads();
            if (H.mode_pw[b] != kHyFloat) {
                gen_hy_minmax_d(tid, gsmh, A, H, b);
                __syncthreads();
                gen_hy_qparams(tid, gsmh, H, tid == 0 ? H.mode_pw[b] : kHyFloat);
                __syncthreads();
                gen_hy_quant_d(tid, gsmh, A, H, b);
                __syncthreads();
                gen_hy_pointwise(tid, gsmh, A, W, H, b);
            } else {
                gen_f32_pointwise(tid, gsmh, A, W, b);
            }
            __syncthreads();
        }
        const int hpos = t % A.head_rows;
        if (H.mode_head != kHyFloat) {
            gen_hy_head_insert(tid, gsmh, A, H, hpos);
            __syncthreads();
            gen_hy_qparams(tid, gsmh, H, tid == 0 ? H.mode_head : kHyFloat);
            __syncthreads();
            gen_hy_quant_head(tid, gsmh, A, H);
            __syncthreads();
            gen_hy_head_partial(tid, gsmh, A, H, hpos);
            __syncthreads();
            gen_hy_head_finish(tid, gsmh, A, W, H, probs + s * probs_stream_stride + t);
        } else {
            gen_f32_head_partial(tid, gsmh, A, W, hpos);
            __syncthreads();
            gen_f32_head_finish(tid, gsmh, A, W, probs + s * probs_stream_stride + t);
        }
        // thread 0's reads of d[] / the quantiser parameters in the head finish are a barrier ahead of their next writers
    }
    gen_f32_tail_gather(tid, gsmh, A, in, n_steps);
    __syncthreads();
    gen_hy_tail_store(tid, gsmh, A, my_state, my_pend, A.ring0 + n_pend + n_rows - A.stride * n_steps, n_steps);
}

__global__ void gen_fill_state_i8_kernel(GenArch A, GenWeightsI8 W, int8_t *__restrict__ state, int8_t *__restrict__ pend,
                                         const int32_t *__restrict__ ids, int n, int n_streams) {
    const long long per = (long long)A.state_elems + (long long)A.pend_cap * kNumChannels;
    const long long total = (long long)n * per;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long k = i / per;
        const int e = (int)(i - k * per);
        const long long s = ids ? ids[k] : k;
        if (s < 0 || s >= n_streams) continue;
        if (e < A.state_elems) state[s * A.state_elems + e] = gen_i8_reset_value(A, W, e);
        else pend[s * (long long)A.pend_cap * kNumChannels + (e - A.state_elems)] = (int8_t)W.zp[0];
    }
}

namespace {
// shared memory above 48 KB is opt-in per function and per device
template <typename K>
cudaError_t allow_smem(K kernel, size_t bytes) {
    if (bytes <= 48 * 1024) return cudaSuccess;
    return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
}
}  // namespace

cudaError_t launch_nn_generic_f32(const GenArch &A, const GenWeightsF32 &W, float *state, float *pend, int n_pend, const void *rows,
                                  long long rows_stream_stride_bytes, int n_rows, int row_type, float *probs, long long probs_stream_stride,
                                  int n_streams, cudaStream_t st) {
    if (n_streams <= 0) return cudaSuccess;
    const size_t smem = (size_t)A.sm_elems * 4;
    cudaError_t e = allow_smem(nn_generic_f32_kernel, smem);
    if (e != cudaSuccess) return e;
    nn_generic_f32_kernel<<<(unsigned)n_streams, kGenThreads, smem, st>>>(A, W, state, pend, n_pend, rows, rows_stream_stride_bytes, n_rows, row_type,
                                                                          probs, probs_stream_stride);
    return cudaGetLastError();
}

cudaError_t launch_nn_generic_i8(const GenArch &A, const GenWeightsI8 &W, int8_t *state, int8_t *pend, int n_pend, const void *rows,
                                 long long rows_stream_stride_bytes, int n_rows, int row_type, float *probs, long long probs_stream_stride,
                                 int n_streams, cudaStream_t st) {
    if (n_streams <= 0) return cudaSuccess;
    const size_t smem = (size_t)A.sm_elems * 4;
    cudaError_t e = allow_smem(nn_generic_i8_kernel, smem);
    if (e != cudaSuccess) return e;
    nn_generic_i8_kernel<<<(unsigned)n_streams, kGenThreads, smem, st>>>(A, W, state, pend, n_pend, rows, rows_stream_stride_bytes, n_rows, row_type,
                                                                         probs, probs_stream_stride);
    return cudaGetLastError();
}

cudaError_t launch_nn_generic_hybrid(const GenArch &A, const GenWeightsF32 &W, const GenHybrid &H, float *state, float *pend, int n_pend,
                                     const void *rows, long long rows_stream_stride_bytes, int n_rows, int row_type, float *probs,
                                     long long probs_stream_stride, int n_streams, cudaStream_t st) {
    if (n_streams <= 0) return cudaSuccess;
    const size_t smem = (size_t)H.sm_elems * 4;
    cudaError_t e = allow_smem(nn_generic_hybrid_kernel, smem);
    if (e != cudaSuccess) return e;
    nn_generic_hybrid_kernel<<<(unsigned)n_streams, kGenThreads, smem, st>>>(A, W, H, state, pend, n_pend, rows, rows_stream_stride_bytes, n_rows,
                                                                             row_type, probs, probs_stream_stride);
    return cudaGetLastError();
}

cudaError_t launch_gen_fill_state_i8(const GenArch &A, const GenWeightsI8 &W, int8_t *state, int8_t *pend, int n, const int32_t *ids, int n_streams,
                                     cudaStream_t st) {
    if (n <= 0) return cudaSuccess;
    const long long total = (long long)n * ((long long)A.state_elems + (long long)A.pend_cap * kNumChannels);
    const unsigned blocks = (unsigned)((total + 255) / 256 < 132 * 16 ? (total + 255) / 256 : 132 * 16);
    gen_fill_state_i8_kernel<<<blocks, 256, 0, st>>>(A, W, state, pend, ids, n, n_streams);
    return cudaGetLastError();
}

}  // namespace mww
