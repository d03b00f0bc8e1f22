// mww_nn_live.cu -- sm_90a kernel + launcher of the live-step MixedNet (one model step for many streams per
// launch; phase functions and rationale: mww_nn_live.cuh).
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <cstdlib>

#include "mww_kernels.h"
#include "mww_nn_live.cuh"

namespace mww {

// persistent CTAs: each walks groups of 32 streams; 1x1 weights are staged once per CTA
__global__ void __launch_bounds__(kLiveThreads, 2)
nn_f32_live_kernel(NnWeightsF32 W, float *__restrict__ state, float *__restrict__ pend, int n_pend, const void *__restrict__ rows,
                   long long rows_stream_stride_bytes, int rows_are_f32, float *__restrict__ probs, long long probs_stride,
                   int n_streams, LiveHeads heads) {
    extern __shared__ __align__(16) float sm[];
    const int tid = threadIdx.x;
    LiveInput in;
    in.state = state; in.pend = pend; in.n_pend = n_pend; in.rows = rows;
    in.rows_stream_stride_bytes = rows_stream_stride_bytes; in.rows_are_f32 = rows_are_f32;
    live_load_weights(tid, sm, W);
    __syncthreads();
    const int n_groups = (n_streams + kLiveStreams - 1) / kLiveStreams;
    for (int g = blockIdx.x; g < n_groups; g += gridDim.x) {
        const long long s0 = (long long)g * kLiveStreams;
        const int n_valid = min(kLiveStreams, n_streams - (int)s0);
        float keep[4][kLiveKeep];
        live_build_a(tid, sm, in, s0, n_valid, keep);
        __syncthreads();
        live_write_tail(tid, state, pend, s0, n_valid, keep);
        live_first_conv_mma(tid, sm, W.w0, 32);
        __syncthreads();
        live_depthwise<0>(tid, sm, W, state, s0, n_valid, heads.h[0]); __syncthreads();
        live_pointwise_mma<0>(tid, sm, W); __syncthreads();
        live_depthwise<1>(tid, sm, W, state, s0, n_valid, heads.h[1]); __syncthreads();
        live_pointwise_mma<1>(tid, sm, W); __syncthreads();
        live_depthwise<2>(tid, sm, W, state, s0, n_valid, heads.h[2]); __syncthreads();
        live_pointwise_mma<2>(tid, sm, W); __syncthreads();
        live_depthwise<3>(tid, sm, W, state, s0, n_valid, heads.h[3]); __syncthreads();
        live_pointwise_mma<3>(tid, sm, W); __syncthreads();
        live_head_partial(tid, sm, W, state, s0, n_valid, heads.h[4]);
        __syncthreads();
        live_head_finish(tid, sm, W, s0, n_valid, probs, probs_stride);
        // the next group's D / H writes are separated from these reads by the barriers at its top
    }
}

// v2 (mww_nn_live.cuh "warp-specialised live step"): threads 0..255 = layer chain, 256..767 = ring streamers
constexpr int kBarChain = 1, kBarFull0 = 2, kBarEmpty0 = 4, kBarAEmpty = 6;   // named barriers: full / empty come in pairs (buffer 0, 1)
__global__ void __launch_bounds__(kLive2Threads, 1)
nn_f32_live2_kernel(NnWeightsF32 W, float *__restrict__ state, float *__restrict__ pend, int n_pend, const void *__restrict__ rows,
                    long long rows_stream_stride_bytes, int rows_are_f32, float *__restrict__ probs, long long probs_stride,
                    int n_streams, LiveHeads heads, int debug_mode) {
    // debug_mode (MWW_LIVE_MODE, timing experiments only -- results are garbage): 1 = streamers skip their loads, 2 = the chain
    // skips its work; both keep the barrier protocol, so the other side runs at its own pace
    extern __shared__ __align__(16) float sm[];
    const int tid = threadIdx.x;
    for (int L = 1; L < 4; ++L) {                                   // 1x1 weights of blocks 1..3, resident for the whole launch
        float *dst = sm + (L == 1 ? kLiveOffPw1 : (L == 2 ? kLiveOffPw2 : kLiveOffPw3));
        for (int e = tid; e < 64 * 64; e += kLive2Threads) dst[(e >> 6) * kWLd + (e & 63)] = W.pw_w[L][e];
    }
    live2_stage_chain_tables(tid, kLive2Threads, sm, W);
    __syncthreads();
    const int n_groups = (n_streams + kLiveStreams - 1) / kLiveStreams;
    LiveInput in;
    in.state = state; in.pend = pend; in.n_pend = n_pend; in.rows = rows;
    in.rows_stream_stride_bytes = rows_stream_stride_bytes; in.rows_are_f32 = rows_are_f32;
    if (tid >= kLive2ChainThreads) {
        // ---- streamers: P of group k into buffer k & 1 (at most two groups ahead of the chain), then the group's first-conv
        // window into A as soon as the chain's first conv of the previous group has let go of it ----
        const int st = tid - kLive2ChainThreads;
        int k = 0;
        for (int g = blockIdx.x; g < n_groups; g += gridDim.x, ++k) {
            const int buf = k & 1;
            if (k >= 2) bar_sync(kBarEmpty0 + buf, kLive2Threads);                  // the chain is done with this P buffer
            const long long s0 = (long long)g * kLiveStreams;
            const int n_valid = min(kLiveStreams, n_streams - (int)s0);
            if (debug_mode != 1) live2_stream_group(st, W, state, s0, n_valid, heads, sm + kLive2OffP + buf * kLive2PFloats);
            if (k >= 1) bar_sync(kBarAEmpty, kLive2Threads);                        // first conv + tail of group k - 1 have read A
            if (debug_mode != 1) live2_build_a<kLive2StreamThreads>(st, sm, in, s0, n_valid);
            bar_arrive(kBarFull0 + buf, kLive2Threads);
        }
        return;
    }
    // ---- chain: shared memory in, ring rows / scores out; no global load on its critical path ----
    int k = 0;
    for (int g = blockIdx.x; g < n_groups; g += gridDim.x, ++k) {
        const int buf = k & 1;
        const float *p_buf = sm + kLive2OffP + buf * kLive2PFloats;
        const long long s0 = (long long)g * kLiveStreams;
        const int n_valid = min(kLiveStreams, n_streams - (int)s0);
        bar_sync(kBarFull0 + buf, kLive2Threads);                                   // P and A of this group are complete
        if (debug_mode == 2) {
            bar_arrive(kBarAEmpty, kLive2Threads);
            bar_arrive(kBarEmpty0 + buf, kLive2Threads);
            continue;
        }
        live_first_conv_mma(tid, sm, sm + kLive2OffW0, kLive2W0Pitch);
        bar_sync(kBarChain, kLive2ChainThreads);                                    // H complete, every warp is done reading A as an operand
        live2_write_tail(tid, sm, in, state, pend, s0, n_valid);                    // new first-conv ring + pending rows, from A
        bar_arrive(kBarAEmpty, kLive2Threads);
        live2_dw_from_p<0>(tid, sm, state, s0, n_valid, heads.h[0], p_buf); bar_sync(kBarChain, kLive2ChainThreads);
        live_pointwise_mma<0, true>(tid, sm, W); bar_sync(kBarChain, kLive2ChainThreads);
        live2_dw_from_p<1>(tid, sm, state, s0, n_valid, heads.h[1], p_buf); bar_sync(kBarChain, kLive2ChainThreads);
        live_pointwise_mma<1, true>(tid, sm, W); bar_sync(kBarChain, kLive2ChainThreads);
        live2_dw_from_p<2>(tid, sm, state, s0, n_valid, heads.h[2], p_buf); bar_sync(kBarChain, kLive2ChainThreads);
        live_pointwise_mma<2, true>(tid, sm, W); bar_sync(kBarChain, kLive2ChainThreads);
        live2_dw_from_p<3>(tid, sm, state, s0, n_valid, heads.h[3], p_buf); bar_sync(kBarChain, kLive2ChainThreads);
        live_pointwise_mma<3, true>(tid, sm, W); bar_sync(kBarChain, kLive2ChainThreads);
        live2_dw_from_p<4>(tid, sm, state, s0, n_valid, heads.h[4], p_buf);
        bar_arrive(kBarEmpty0 + buf, kLive2Threads);                                // last read of this P buffer
        bar_sync(kBarChain, kLive2ChainThreads);
        live_head_finish_b(tid, sm, sm[kLive2OffSmall + kLive2SmallHeadBias], s0, n_valid, probs, probs_stride);
        bar_sync(kBarChain, kLive2ChainThreads);                                    // D is rewritten by the next group
    }
}

// =====================================================================================================================
// v3: the ring data arrive by bulk copy (TMA) instead of register loads.  In v2 the two halves together take much longer than
// either alone (MWW_LIVE_MODE runs one half): the chain's shared-memory operands and the streamers' global loads queue in the
// same LSU / L1 miss pipeline.  Here one elected thread issues one
// cp.async.bulk (global -> shared, 16 384 B = rings 1..5 of one stream, contiguous in the state layout) per stream into a
// ring of four stages; nine "P" warps (one ring column per thread, its R rotated taps in registers) turn each stage into the
// stream's 288 partial sums; six warps build the first-conv window one group ahead; the 8 chain warps are v2's.
// P is single-buffered: a P thread keeps the 32 sums of the NEXT group in registers and writes them once the chain's layer of
// the current group has read the buffer (one full / empty named-barrier pair per ring) -- the second P buffer of v2 became
// two more stages (bytes in flight are what an HBM-bound kernel is made of).
// The sums and their order are v2's (= v1's): the three kernels are bit-identical.
constexpr int kLive3PThreads = kLive2Cols;                            // 288: one thread per ring column
constexpr int kLive3AThreads = kLive3WindowThreads;
constexpr int kLive3Threads = kLive2ChainThreads + kLive3PThreads + kLive3AThreads + 32;   // + the producer's warp
constexpr int kLive3PBase = kLive2ChainThreads, kLive3ABase = kLive3PBase + kLive3PThreads, kLive3ProdBase = kLive3ABase + kLive3AThreads;
constexpr int kLive3StageFloats = kStateFloats - kStateOff[1];        // rings 1..5 of one stream
constexpr int kLive3Stages = 4;
constexpr int kLive3OffStageLo = kLive2OffW0;                         // stages 0, 1: where v2 keeps the first-conv weights (v3 reads them from L2)
constexpr int kLive3OffStageHi = kLive2OffP + kLive2PFloats;          // stages 2, 3: v2's second P buffer
constexpr int kLive3OffMbar = kLive3OffStageLo + 2 * kLive3StageFloats;
constexpr int kLive3SmemBytes = (kLive3OffMbar + 4 * kLive3Stages) * 4;
static_assert(kLive3StageFloats == 4096 && (kLive3StageFloats * 4) % 16 == 0 && (kStateOff[1] * 4) % 16 == 0 && (kStateFloats * 4) % 16 == 0,
              "bulk copy granularity");
static_assert((kLive3OffStageHi * 4) % 128 == 0 && 2 * kLive3StageFloats <= kLive2PFloats, "stages 2, 3 fit the second P buffer");
static_assert(kLive3SmemBytes <= 232448, "shared memory per CTA");
static_assert(kLive3PThreads / 32 == 9 && kLiveStreams % kLive3Stages == 0 && (kLiveStreams / kLive3Stages) % 2 == 0,
              "P warps 1 + 2 + 2 + 2 + 2; stage index and parity of a stream are compile-time");
__host__ __device__ constexpr int live3_stage_off(int s) { return s < 2 ? kLive3OffStageLo + s * kLive3StageFloats : kLive3OffStageHi + (s - 2) * kLive3StageFloats; }
// named barriers of v3
constexpr int kBar3Chain = 1, kBar3AFull = 2, kBar3AEmpty = 3, kBar3RingFull = 4, kBar3RingEmpty = 9, kBar3Window = 14;
__host__ __device__ constexpr int live3_ring_count(int i) { return kLive2ChainThreads + live_ring_cols(i); }

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *b, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *b) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(b)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *b, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *b, unsigned parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "W: mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra D;\n\tbra W;\n\tD:\n\t}" ::"r"(smem_u32(b)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, unsigned bytes, uint64_t *b) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
                 "l"(__cvta_generic_to_global(src)), "r"(bytes), "r"(smem_u32(b))
                 : "memory");
}

// one P warp's whole life: ring I, column c of it
template <int I>
__device__ __forceinline__ void live3_p_warp(int c, int lane, float *sm, uint64_t *full, uint64_t *empty, const NnWeightsF32 &W, int head,
                                             int n_groups, int debug_mode) {
    constexpr int R = live_ring_rows(I);
    constexpr int per_group = kLiveStreams / kLive3Stages;             // uses of each stage per group (even: parity restarts every group)
    float w[R], bias;
    live3_p_taps<I>(W, c, head, w, bias);
    float *p_col = sm + kLive2OffP + (live2_col_base(I) + c) * kLive2PPitch;
    int k = 0;
    for (int g = blockIdx.x; g < n_groups; g += gridDim.x, ++k) {
        // 32 sums per thread stay in registers until the chain lets go of the P buffer.  The stream loop is rolled (8 rounds of
        // kLive3Stages streams; unrolled it was 93 KB of code over the five instances and `no_inst` led the chain's stall
        // samples): each round shifts the register file by one round and appends, so indices stay compile-time.
        float acc[kLiveStreams];
        if (debug_mode != 1) {
#pragma unroll 1
            for (int round = 0; round < per_group; ++round) {
#pragma unroll
                for (int i = 0; i < kLiveStreams - kLive3Stages; ++i) acc[i] = acc[i + kLive3Stages];
#pragma unroll
                for (int s = 0; s < kLive3Stages; ++s) {
                    mbar_wait(full + s, (unsigned)(round & 1));
                    acc[kLiveStreams - kLive3Stages + s] = live3_p_sum<I>(sm + live3_stage_off(s), c, w, bias);
                    __syncwarp();
                    if (lane == 0) mbar_arrive(empty + s);
                }
            }
        } else {
#pragma unroll
            for (int sl = 0; sl < kLiveStreams; ++sl) acc[sl] = bias;
        }
        if (k >= 1) bar_sync(kBar3RingEmpty + I, live3_ring_count(I));                   // the chain's layer I of group k - 1 has read P
#pragma unroll
        for (int sl = 0; sl < kLiveStreams; ++sl) p_col[sl] = acc[sl];
        bar_arrive(kBar3RingFull + I, live3_ring_count(I));
    }
}

__global__ void __launch_bounds__(kLive3Threads, 1)
nn_f32_live3_kernel(NnWeightsF32 W, float *__restrict__ state, float *__restrict__ pend, int n_pend, const void *__restrict__ rows,
                    long long rows_stream_stride_bytes, int rows_are_f32, float *__restrict__ probs, long long probs_stride,
                    int n_streams, LiveHeads heads, int debug_mode) {
    extern __shared__ __align__(16) float sm[];
    const int tid = threadIdx.x;
    for (int L = 1; L < 4; ++L) {
        float *dst = sm + (L == 1 ? kLiveOffPw1 : (L == 2 ? kLiveOffPw2 : kLiveOffPw3));
        for (int e = tid; e < 64 * 64; e += kLive3Threads) dst[(e >> 6) * kWLd + (e & 63)] = W.pw_w[L][e];
    }
    live2_stage_chain_tables(tid, kLive3Threads, sm, W, false);
    uint64_t *full = reinterpret_cast<uint64_t *>(sm + kLive3OffMbar), *empty = full + kLive3Stages;
    if (tid == 0) {
        for (int s = 0; s < kLive3Stages; ++s) { mbar_init(full + s, 1); mbar_init(empty + s, kLive3PThreads / 32); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const int n_groups = (n_streams + kLiveStreams - 1) / kLiveStreams;
    LiveInput in;
    in.state = state; in.pend = pend; in.n_pend = n_pend; in.rows = rows;
    in.rows_stream_stride_bytes = rows_stream_stride_bytes; in.rows_are_f32 = rows_are_f32;
    if (tid >= kLive3ProdBase) {
        // ---- producer: one bulk copy per stream, as far ahead as the stages allow ----
        if (tid != kLive3ProdBase || debug_mode == 1) return;
        unsigned n = 0;
        constexpr int ring1 = kStateOff[1];
        for (int g = blockIdx.x; g < n_groups; g += gridDim.x) {
            const long long s0 = (long long)g * kLiveStreams;
            const int n_valid = min(kLiveStreams, n_streams - (int)s0);
            for (int sl = 0; sl < kLiveStreams; ++sl, ++n) {
                const unsigned s = n % kLive3Stages, use = n / kLive3Stages;
                if (use >= 1) mbar_wait(empty + s, (use - 1) & 1u);
                const long long stream = s0 + min(sl, n_valid - 1);          // a short last group re-reads its last stream; the chain masks it
                mbar_expect_tx(full + s, kLive3StageFloats * 4);
                bulk_g2s(sm + live3_stage_off((int)s), state + (size_t)stream * kStateFloats + ring1, kLive3StageFloats * 4, full + s);
            }
        }
        return;
    }
    if (tid >= kLive3ABase) {
        // ---- first-conv window of group k into A as soon as the chain's first conv of group k - 1 has let go of it ----
        const int at = tid - kLive3ABase;
        float v[kLive3WindowPerThread];
        int k = 0;
        auto load = [&](int gl) {
            const long long s0 = (long long)gl * kLiveStreams;
            const int n_valid = min(kLiveStreams, n_streams - (int)s0);
            live3_window_load(at, in, s0, n_valid, v);
            if (n_pend != 0) {
                bar_sync(kBar3Window, kLive3AThreads);                             // every old pending row of the group has been read
                live3_pend_store(at, in, pend, s0, n_valid);
            }
        };
        if ((int)blockIdx.x < n_groups && debug_mode != 1) load((int)blockIdx.x);
        for (int g = blockIdx.x; g < n_groups; g += gridDim.x, ++k) {
            if (k >= 1) bar_sync(kBar3AEmpty, kLive2ChainThreads + kLive3AThreads);
            if (debug_mode != 1) live3_window_store(at, sm, v);
            bar_arrive(kBar3AFull, kLive2ChainThreads + kLive3AThreads);
            const int gn = g + (int)gridDim.x;
            if (gn < n_groups && debug_mode != 1) load(gn);                        // the next group's window, a chain period early
        }
        return;
    }
    if (tid >= kLive3PBase) {
        const int pt = tid - kLive3PBase, pw = pt >> 5, lane = pt & 31;
        if (pw == 0) live3_p_warp<0>(pt, lane, sm, full, empty, W, heads.h[0], n_groups, debug_mode);
        else if (pw <= 2) live3_p_warp<1>(pt - 32, lane, sm, full, empty, W, heads.h[1], n_groups, debug_mode);
        else if (pw <= 4) live3_p_warp<2>(pt - 96, lane, sm, full, empty, W, heads.h[2], n_groups, debug_mode);
        else if (pw <= 6) live3_p_warp<3>(pt - 160, lane, sm, full, empty, W, heads.h[3], n_groups, debug_mode);
        else live3_p_warp<4>(pt - 224, lane, sm, full, empty, W, heads.h[4], n_groups, debug_mode);
        return;
    }
    // ---- chain (v2's, with the first conv's B fragments from L2 like v1) ----
    const float *p_buf = sm + kLive2OffP;
    for (int g = blockIdx.x; g < n_groups; g += gridDim.x) {
        const long long s0 = (long long)g * kLiveStreams;
        const int n_valid = min(kLiveStreams, n_streams - (int)s0);
        bar_sync(kBar3AFull, kLive2ChainThreads + kLive3AThreads);                  // the window of this group is complete
        if (debug_mode == 2) {
            bar_arrive(kBar3AEmpty, kLive2ChainThreads + kLive3AThreads);
            for (int i = 0; i < 5; ++i) {
                bar_sync(kBar3RingFull + i, live3_ring_count(i));
                bar_arrive(kBar3RingEmpty + i, live3_ring_count(i));
            }
            continue;
        }
        live_first_conv_mma(tid, sm, W.w0, 32);
        bar_sync(kBar3Chain, kLive2ChainThreads);
        live3_write_ring0(tid, sm, state, s0, n_valid);
        bar_arrive(kBar3AEmpty, kLive2ChainThreads + kLive3AThreads);
#define MWW_LIVE3_LAYER(I)                                                                         \
        bar_sync(kBar3RingFull + I, live3_ring_count(I));                                          \
        live2_dw_from_p<I>(tid, sm, state, s0, n_valid, heads.h[I], p_buf);                        \
        bar_arrive(kBar3RingEmpty + I, live3_ring_count(I));                                       \
        bar_sync(kBar3Chain, kLive2ChainThreads);
        MWW_LIVE3_LAYER(0) live_pointwise_mma<0, true>(tid, sm, W); bar_sync(kBar3Chain, kLive2ChainThreads);
        MWW_LIVE3_LAYER(1) live_pointwise_mma<1, true>(tid, sm, W); bar_sync(kBar3Chain, kLive2ChainThreads);
        MWW_LIVE3_LAYER(2) live_pointwise_mma<2, true>(tid, sm, W); bar_sync(kBar3Chain, kLive2ChainThreads);
        MWW_LIVE3_LAYER(3) live_pointwise_mma<3, true>(tid, sm, W); bar_sync(kBar3Chain, kLive2ChainThreads);
        MWW_LIVE3_LAYER(4)
#undef MWW_LIVE3_LAYER
        live_head_finish_b(tid, sm, sm[kLive2OffSmall + kLive2SmallHeadBias], s0, n_valid, probs, probs_stride);
        bar_sync(kBar3Chain, kLive2ChainThreads);
    }
}

cudaError_t launch_nn_f32_live(const NnWeightsF32 &W, float *state, float *pend, int n_pend, const void *rows,
                               long long rows_stream_stride_bytes, int rows_are_f32, float *probs, long long probs_stride,
                               int n_streams, const LiveHeads &heads, int sm_count, int variant, cudaStream_t st) {
    if (n_streams <= 0) return cudaSuccess;
    static bool attr_done[64] = {};
    const bool v1 = variant != 2 && variant != 3;   // 2 = warp-specialised with register loads, 3 = with bulk copies (MWW_LIVE_VARIANT at mww_create)
    static const int debug_mode = getenv("MWW_LIVE_MODE") ? atoi(getenv("MWW_LIVE_MODE")) : 0;
    if (first_launch_on_this_device(attr_done)) {
        cudaError_t e = cudaFuncSetAttribute(nn_f32_live_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kLiveSmemBytes);
        if (e == cudaSuccess) e = cudaFuncSetAttribute(nn_f32_live2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kLive2SmemBytes);
        if (e == cudaSuccess) e = cudaFuncSetAttribute(nn_f32_live3_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kLive3SmemBytes);
        if (e != cudaSuccess) return e;
    }
    const int n_groups = (n_streams + kLiveStreams - 1) / kLiveStreams;
    if (v1) {
        const int grid = std::min(n_groups, 2 * sm_count);
        nn_f32_live_kernel<<<grid, kLiveThreads, kLiveSmemBytes, st>>>(W, state, pend, n_pend, rows, rows_stream_stride_bytes, rows_are_f32, probs,
                                                                       probs_stride, n_streams, heads);
    } else if (variant == 3) {
        const int grid = std::min(n_groups, sm_count);
        nn_f32_live3_kernel<<<grid, kLive3Threads, kLive3SmemBytes, st>>>(W, state, pend, n_pend, rows, rows_stream_stride_bytes, rows_are_f32, probs,
                                                                          probs_stride, n_streams, heads, debug_mode);
    } else {
        const int grid = std::min(n_groups, sm_count);
        nn_f32_live2_kernel<<<grid, kLive2Threads, kLive2SmemBytes, st>>>(W, state, pend, n_pend, rows, rows_stream_stride_bytes, rows_are_f32, probs,
                                                                          probs_stride, n_streams, heads, debug_mode);
    }
    return cudaGetLastError();
}

__global__ void nn_live_canonicalise_kernel(float *__restrict__ state, int n_streams, LiveHeads heads) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (long long)n_streams * 288) return;
    live_canonicalise_column(state, e / 288, (int)(e % 288), heads);
}

cudaError_t launch_nn_live_canonicalise(float *state, int n_streams, const LiveHeads &heads, cudaStream_t st) {
    if (n_streams <= 0) return cudaSuccess;
    const long long total = (long long)n_streams * 288;
    nn_live_canonicalise_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(state, n_streams, heads);
    return cudaGetLastError();
}

}  // namespace mww
