// mww_nn_tc.cu -- fp32 streaming MixedNet, clip formulation, on the Hopper warpgroup tensor cores (wgmma).
//
// Same graph and ring semantics as mww_nn_dev.cuh / mww_nn.cu (microwakeword/mixednet.py:307-386, layers/stream.py:581-595,
// one call = inference.py:109-123 for many steps); what changes is how the dense 88 % of the MACs -- the strided first conv
// (K = 200) and the four 1x1 projections -- are contracted:
//
//   * one CTA owns one stream and a chunk of up to 128 MODEL STEPS: time is the M dimension; each of the CTA's two warpgroups
//     contracts 64 of the steps (wgmma M = 64);
//   * the CUDA cores produce each contraction's A operand (im2col of the feature rows / the depthwise MixConv output) ONCE, already
//     split for 3xTF32 into a hi and a lo plane, in the layout the tensor core reads: K cut into slots of 32 values = 128 bytes,
//     a slot = [128 steps][128 B] with the hardware's 128-byte XOR swizzle, so a warp whose lanes are 32 consecutive channels of
//     one step stores 128 contiguous bytes (no bank conflicts);
//   * the weights are split and laid out the same way once, at mww_create (build_tc_weights), and stream from L2 into shared memory
//     with 16-byte cp.async one layer ahead of their use;
//   * both warpgroups issue wgmma.mma_async.m64nNk8.f32.tf32.tf32 with A and B through shared-memory matrix descriptors: per K = 8
//     step the three 3xTF32 products lo*hi, hi*lo, hi*hi accumulate into the same fp32 register tile [64 steps x N];
//   * the epilogue takes the accumulator straight from the registers, adds the folded-BatchNorm bias, applies ReLU and writes the
//     next layer's activations [channel][time] for the depthwise stage.
// Depthwise taps, ring buffers, the 17-row head and the sigmoid stay on CUDA cores, in shared memory for the whole call.
//
// The mma.sync kernel (mww_nn.cu) remains the path for float32 feature rows and for calls shorter than kTcMinSteps steps.
#include <cuda_runtime.h>
#include <cstdlib>
#include <cstring>

#include <type_traits>
#include <vector>

#include "mww_kernels.h"
#include "mww_nn_tc.h"
#include "mww_nn_tc_prep.h"

namespace mww {

namespace {

constexpr int kTcThreads = 256;
constexpr int kTcM = 128;                       // model steps per chunk = MMA M
constexpr int kLdx = 151;                       // activation buffer pitch [channel][22 history + 128 steps + 1]: odd -> conflict-free
constexpr int kFeatRows = 3 * kTcM + 2;         // feature rows one chunk's first conv can touch

// ---- shared memory map (bytes): 102.6 KB, TWO CTAs per SM -- a stream's layer chain is strictly serial (produce -> MMA -> epilogue ->
// next layer), so the only way to keep the SM busy is a second, independent stream.  Every contraction is therefore fed ONE K-slot
// (32 input channels) at a time:
constexpr int kOffA = 0;                        // one K-slot of A: hi plane 16 KB + lo plane 16 KB
constexpr int kAPlaneBytes = 16384;
constexpr int kOffB = 32768;                    // two K-slots of B (double buffer): [N <= 64 rows][128 B] hi + lo = 16 KB each
constexpr int kBSlotBytes = 16384;
constexpr int kOffX = kOffB + 2 * kBSlotBytes;  // activations [64][kLdx]; the chunk's raw uint16 feature rows alias it during the first conv
constexpr int kOffSmall = kOffX + 64 * kLdx * 4;   // first-conv ring rows -2, -1 and the pending rows as floats [4][40]
constexpr int kTcSmemBytes = kOffSmall + 4 * kNumChannels * 4;
static_assert(2 * (kTcSmemBytes + 1024) <= 232448, "two CTAs per SM");
static_assert(kFeatRows * kNumChannels * 2 <= 64 * kLdx * 4, "feature rows alias the activation buffer");
static_assert(kOffA % 1024 == 0 && kOffB % 1024 == 0, "swizzled operand slots need 1024-byte alignment");

// 128-byte-swizzled K-major slot: sw128_off(row, kk), mww_nn_tc_prep.h
__device__ __forceinline__ void split_tf32f(float x, float &hi, float &lo) {
    hi = __uint_as_float(__float_as_uint(x) & 0xFFFFE000u);
    lo = x - hi;
}
// element (step t, position kk in the K-slot) of the A operand: hi and lo plane
__device__ __forceinline__ void store_split(unsigned char *a_base, int t, int kk, float v) {
    float hi, lo;
    split_tf32f(v, hi, lo);
    unsigned char *p = a_base + sw128_off(t, kk);
    *reinterpret_cast<float *>(p) = hi;
    *reinterpret_cast<float *>(p + kAPlaneBytes) = lo;
}

// wgmma shared-memory matrix descriptor of a K-major operand with the 128-byte swizzle
__device__ __forceinline__ uint64_t desc_sw128(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);      // start address
    d |= (uint64_t)1 << 16;                           // leading byte offset (unused: the operand is one swizzle atom wide in K)
    d |= (uint64_t)(1024 >> 4) << 32;                 // stride byte offset: next group of 8 rows
    d |= (uint64_t)1 << 62;                           // SWIZZLE_128B
    return d;
}
// D[64 x N] (+)= A[64 x 8] B[8 x N], tf32 operands from shared memory, fp32 accumulator in the warpgroup's registers: N / 2 per thread
template <int N_>
__device__ __forceinline__ void mma_tf32(float (&d)[32], uint64_t da, uint64_t db, int accumulate);
template <>
__device__ __forceinline__ void mma_tf32<32>(float (&d)[32], uint64_t da, uint64_t db, int accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
                 "%16, %17, p, 1, 1;\n\t}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
                   "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                 : "l"(da), "l"(db), "r"(accumulate));
}
template <>
__device__ __forceinline__ void mma_tf32<64>(float (&d)[32], uint64_t da, uint64_t db, int accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
                 "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
                   "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
                   "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
                   "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "l"(da), "l"(db), "r"(accumulate));
}
// the accumulator registers are ordered against the asynchronous MMAs: neither side of a fence / wait may be moved across it
__device__ __forceinline__ void fence_acc(float (&d)[32]) {
#pragma unroll
    for (int i = 0; i < 32; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// one K-slot for this warpgroup's 64 steps: KSTEPS K = 8 steps (4, or 1 for the tail of the first conv) of the three 3xTF32 products;
// A rows at a_s (lo plane at +16 KB), B slot at b_s with its lo plane `b_plane` bytes further.  Returns with the MMAs complete.
template <int N_, int KSTEPS>
__device__ __forceinline__ void issue_slot(float (&d)[32], uint32_t a_s, uint32_t b_s, uint32_t b_plane, bool clears) {
    fence_acc(d);
    asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory");
#pragma unroll
    for (int ks = 0; ks < KSTEPS; ++ks) {
        const uint32_t a_hi = a_s + (uint32_t)ks * 32, a_lo = a_hi + kAPlaneBytes;
        const uint32_t b_hi = b_s + (uint32_t)ks * 32, b_lo = b_hi + b_plane;
        mma_tf32<N_>(d, desc_sw128(a_lo), desc_sw128(b_hi), !(clears && ks == 0));
        mma_tf32<N_>(d, desc_sw128(a_hi), desc_sw128(b_lo), 1);
        mma_tf32<N_>(d, desc_sw128(a_hi), desc_sw128(b_hi), 1);
    }
    asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory");
    asm volatile("wgmma.wait_group.sync.aligned 0;\n" ::: "memory");
    fence_acc(d);
}
// everything the generic proxy wrote to shared memory (st.shared, completed cp.async) becomes visible to the tensor core
__device__ __forceinline__ void publish_operands() {
    asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
    __syncthreads();
}
__device__ __forceinline__ void cp16(void *smem_dst, const void *gmem_src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((unsigned)__cvta_generic_to_shared(smem_dst)), "l"(gmem_src));
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N_>
__device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N_) : "memory"); }

// ---- geometry of the five ring-carrying activation tensors (inputs of block 0..3 and of the head): channels, ring rows ----
__device__ __forceinline__ constexpr int tc_cin(int i) { return i == 0 ? 32 : 64; }
__device__ __forceinline__ constexpr int tc_ring(int i) { return i == 0 ? 4 : (i == 1 ? 10 : (i == 2 ? 14 : (i == 3 ? 22 : 16))); }

// ring i (HBM layout [row][channel], oldest first; read straight from the stream's state, coalesced) -> history columns [0, R) of X
template <int I>
__device__ __forceinline__ void ring_to_x(int tid, float *x, const float *ring_store) {
    constexpr int R = tc_ring(I), C = tc_cin(I);
    const float *src = ring_store + kStateOff[I + 1];
    for (int e = tid; e < R * C; e += kTcThreads) {
        const int r = e / C, c = e - r * C;
        x[c * kLdx + r] = src[e];
    }
}
// the last R columns of (history ++ n new outputs) become the ring for the next chunk / call
template <int I>
__device__ __forceinline__ void x_to_ring(int tid, const float *x, float *ring_store, int n) {
    constexpr int R = tc_ring(I), C = tc_cin(I);
    float *dst = ring_store + kStateOff[I + 1];
    for (int e = tid; e < R * C; e += kTcThreads) {
        const int r = e / C, c = e - r * C;
        dst[e] = x[c * kLdx + n + r];
    }
}

// depthwise MixConv of block L over X (history + chunk) -> A operand (hi / lo planes), bias included.
// thread -> (channel, time segment); a warp's lanes are 32 consecutive channels of one time step: X reads and A stores conflict-free
template <int L, int K>
__device__ __forceinline__ void depthwise_k(int c, int t0, int t1, const float *x, unsigned char *a_base, const NnWeightsF32 &W) {
    constexpr int R = tc_ring(L), C = tc_cin(L), KMAX = R + 1;
    float w[K];
#pragma unroll
    for (int j = 0; j < K; ++j) w[j] = W.dw_w[L][(KMAX - K + j) * C + c];      // shorter MixConv kernels are zero padded at the front
    const float bias = W.dw_b[L][c];
    const float *xc = x + c * kLdx + (R - (K - 1));                             // output step t reads columns t .. t + K - 1 from here
    constexpr int TN = 8;
    for (int tb = t0; tb < t1; tb += TN) {
        float acc[TN];
#pragma unroll
        for (int i = 0; i < TN; ++i) acc[i] = bias;
#pragma unroll
        for (int i = 0; i < TN + K - 1; ++i) {
            const float xv = xc[tb + i];
#pragma unroll
            for (int tt = 0; tt < TN; ++tt) {
                const int j = i - tt;
                if (j >= 0 && j < K) acc[tt] = fmaf(w[j], xv, acc[tt]);
            }
        }
#pragma unroll
        for (int i = 0; i < TN; ++i) store_split(a_base, tb + i, c & 31, acc[i]);
    }
}
// K-slot H of block L = its input channels 32 H .. 32 H + 31 -- for the two-kernel MixConv blocks exactly one kernel size per slot.
// thread -> (channel 32 H + tid % 32, time segment tid / 32 of 16 steps)
template <int L, int H>
__device__ __forceinline__ void depthwise_slot(int tid, int n, const float *x, unsigned char *a_base, const NnWeightsF32 &W) {
    const int t0 = 16 * (tid >> 5);
    if (t0 >= n) return;                                     // steps beyond the chunk are never read back
    const int t1 = min(t0 + 16, (n + 7) & ~7);
    constexpr int K = L == 0 ? 5 : (L == 1 ? (H == 0 ? 7 : 11) : (L == 2 ? (H == 0 ? 9 : 15) : 23));
    depthwise_k<L, K>(32 * H + (tid & 31), t0, t1, x, a_base, W);
}

// accumulator [128 steps x N] -> (+ bias) ReLU -> X[o][hist + t] for t < n.  wgmma's fragment of warp w of warpgroup g: steps
// 64 g + 16 (w % 4) + lane / 4 (+ 8), columns 8 j + 2 (lane % 4) (+ 1) in d[4 j + 2 h + e]
template <int N_, int HIST>
__device__ __forceinline__ void epilogue(int tid, int n, const float (&d)[32], float *x, const float *bias /* nullptr: none */) {
    const int lane = tid & 31;
    const int t0 = 64 * (tid >> 7) + 16 * ((tid >> 5) & 3) + (lane >> 2);
    if (t0 - (lane >> 2) >= n) return;                        // warp-uniform: this warp's 16 steps are all beyond the chunk
#pragma unroll
    for (int j = 0; j < N_ / 8; ++j) {
        const int c = 8 * j + 2 * (lane & 3);
        const float2 b2 = bias ? __ldg(reinterpret_cast<const float2 *>(bias + c)) : make_float2(0.f, 0.f);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int t = t0 + 8 * h;
            if (t < n) {
                const float r0 = d[4 * j + 2 * h] + b2.x, r1 = d[4 * j + 2 * h + 1] + b2.y;
                x[c * kLdx + HIST + t] = r0 > 0.f ? r0 : 0.f;
                x[(c + 1) * kLdx + HIST + t] = r1 > 0.f ? r1 : 0.f;
            }
        }
    }
}

}  // namespace

// grid = min(streams, 2 x SMs) persistent CTAs (two per SM); 256 threads; one stream at a time, chunks of up to 128 model steps
__global__ void __launch_bounds__(kTcThreads, 2)
nn_f32_clip_tc_kernel(NnWeightsF32 W, TcWeights TW, float *__restrict__ state, float *__restrict__ pend, int n_pend, const uint16_t *__restrict__ rows,
                      long long rows_stream_stride, int n_rows, float *__restrict__ probs, long long probs_stream_stride, int n_streams) {
    extern __shared__ __align__(1024) unsigned char smem[];
    unsigned char *a_base = smem + kOffA, *b_base = smem + kOffB;
    float *x = reinterpret_cast<float *>(smem + kOffX);
    uint16_t *feat = reinterpret_cast<uint16_t *>(smem + kOffX);          // alias: dead before X's first write of a chunk
    float *small = reinterpret_cast<float *>(smem + kOffSmall);           // [0,80): first-conv ring rows -2, -1; [80,160): pending rows
    const int tid = threadIdx.x, wg = tid >> 7;
    // this warpgroup's 64 rows of the A slot (8 KB, a whole number of 1024-byte swizzle atoms)
    const uint32_t a_s = (uint32_t)__cvta_generic_to_shared(a_base) + (uint32_t)wg * 64 * 128, b_s = (uint32_t)__cvta_generic_to_shared(b_base);
    float acc[32];

    // The 14 K-slots of a chunk, in order: first conv 0..6 (N = 32; the last holds K = 8), block 0 (one slot), blocks 1..3 (two each).
    // Slot i's weights sit in B buffer i % 2 and are fetched while slot i - 1 is produced and contracted.
    auto b_src = [&](int i) -> const unsigned char * {
        if (i < 7) return TW.fc + (size_t)i * 8192;
        if (i == 7) return TW.pw[0];
        return TW.pw[(i - 6) >> 1] + (size_t)((i - 8) & 1) * kBSlotBytes;
    };
    auto stage_slot = [&](int i) {
        if (i < 14) {
            const int bytes = i < 7 ? 8192 : kBSlotBytes;
            const unsigned char *src = b_src(i);
            unsigned char *dst = b_base + (i & 1) * kBSlotBytes;
            for (int e = tid * 16; e < bytes; e += kTcThreads * 16) cp16(dst + e, src + e);
        }
        cp_commit();                                     // one group per call (possibly empty): wait_group counts stay uniform
    };
    // after slot i's A operand is in shared memory: its weights have landed -> publish -> each warpgroup contracts its 64 steps (a
    // warpgroup whose steps all lie beyond the chunk skips) -> once both are done with A and B buffer i % 2, prefetch slot i + 2's weights
    auto contract_slot = [&](auto n_out, auto ksteps, int i, int n, bool clears) {
        cp_wait<1>();                                    // all but the most recent group: slot i's weights are here
        publish_operands();
        if (64 * wg < n)
            issue_slot<decltype(n_out)::value, decltype(ksteps)::value>(acc, a_s, b_s + (uint32_t)(i & 1) * kBSlotBytes, i < 7 ? 4096u : 8192u,
                                                                         clears);
        __syncthreads();                                 // A and B buffer i % 2 are free again; the accumulator holds slots <= i
        stage_slot(i + 2);
    };
    using N32 = std::integral_constant<int, 32>;
    using N64 = std::integral_constant<int, 64>;
    using K4 = std::integral_constant<int, 4>;
    using K1 = std::integral_constant<int, 1>;

    const int n_virtual = n_pend + n_rows;
    const int n_steps = n_virtual / 3;
    for (long long s = blockIdx.x; s < n_streams; s += gridDim.x) {
        float *my_state = state + s * kStateFloats;
        float *my_pend = pend + s * 2 * kNumChannels;
        const uint16_t *my_rows = rows + s * rows_stream_stride;
        if (tid < 80) small[tid] = my_state[tid];
        else if (tid < 160) small[tid] = my_pend[tid - 80];
        if (tid == 192) {
            // this stream's rings are read layer by layer further down, the NEXT stream's state and rows one stream from now: ask the L2
            // for them now (bulk prefetch: no registers, nothing to wait for)
            asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(my_state), "r"(kStateFloats * 4) : "memory");
            const long long sn = s + gridDim.x;
            if (sn < n_streams) {
                asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(state + sn * kStateFloats), "r"(kStateFloats * 4) : "memory");
                const unsigned bytes = (unsigned)min((long long)n_rows * kNumChannels * 2, 65536ll) & ~15u;
                if (bytes) asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(rows + sn * rows_stream_stride), "r"(bytes) : "memory");
            }
        }
        for (int step0 = 0; step0 < n_steps; step0 += kTcM) {
            const int n = min(kTcM, n_steps - step0);
            // virtual rows of this chunk: vr0 .. vr0 + 3 n + 2, with vr = -2, -1 the first-conv ring, [0, n_pend) pending, then the call's rows
            const int vr0 = 3 * step0 - 2;
            const int row_lo = max(vr0 - n_pend, 0), row_hi = min(vr0 + 3 * n + 2 - n_pend, n_rows);       // rows of `my_rows` the chunk reads
            {
                const int n16 = (row_hi - row_lo) * (kNumChannels * 2 / 16);                               // 5 x 16 bytes per row
                const unsigned char *src = reinterpret_cast<const unsigned char *>(my_rows + (long long)row_lo * kNumChannels);
                for (int e = tid; e < n16; e += kTcThreads) cp16(reinterpret_cast<unsigned char *>(feat) + 16 * e, src + 16 * e);
                cp_commit();
            }
            stage_slot(0);
            stage_slot(1);
            cp_wait<2>();                                                  // the feature rows (oldest group) are here
            __syncthreads();
            auto feature = [&](int vr, int f) -> float {                  // inference.py:93-94 scaling of raw uint16 rows
                if (vr < 0) return small[(2 + vr) * kNumChannels + f];
                if (vr < n_pend) return small[80 + vr * kNumChannels + f];
                return (float)feat[(vr - n_pend - row_lo) * kNumChannels + f] * kFeatureScale;
            };
            // ---- first conv: K = 200 as seven K-slots accumulated in registers; thread -> (k column tid % 32, steps tid / 32 + 8 i) ----
#pragma unroll 1
            for (int slot = 0; slot < 7; ++slot) {
                const int kk = tid & 31, k = 32 * slot + kk;
                const int j = k / kNumChannels, f = k - j * kNumChannels;
                if (k < 200) {                                             // slot 6 only has the K = 8 step 192..199
                    // steps 0 and 1 of a call's first chunk can touch the first-conv ring / the pending rows; every other element is a raw
                    // uint16 row of this call at an index affine in t: one 16-bit load, convert, scale, split, two stores
                    const int t_pad = (n + 7) & ~7;
                    int t = tid >> 5;
                    for (; t < 2 && t < t_pad; t += 8) store_split(a_base, t, kk, t < n ? feature(vr0 + 3 * t + j, f) : 0.f);
                    const uint16_t *src = feat + (vr0 + j - n_pend - row_lo) * kNumChannels + f;
                    for (; t < n; t += 8) store_split(a_base, t, kk, (float)src[3 * kNumChannels * t] * kFeatureScale);
                    for (; t < t_pad; t += 8) store_split(a_base, t, kk, 0.f);
                }
                if (slot < 6) contract_slot(N32{}, K4{}, slot, n, slot == 0);
                else contract_slot(N32{}, K1{}, slot, n, false);
            }
            // first conv epilogue: ReLU, no bias -> X (block 0's input), its ring history in front.  The feature rows under X are dead.
            ring_to_x<0>(tid, x, my_state);
            epilogue<32, 4>(tid, n, acc, x, nullptr);
            __syncthreads();
            // ---- four MixConv blocks: per K-slot depthwise -> contract; then ring out / next history in / epilogue ----
#define MWW_TC_BLOCK_END(L)                                                                                                                 \
            x_to_ring<L>(tid, x, my_state, n);                          /* the last R columns of (history ++ outputs): the ring for later */ \
            __syncthreads();                                                                                                                \
            ring_to_x<L + 1>(tid, x, my_state);                                                                                             \
            epilogue<64, tc_ring(L + 1)>(tid, n, acc, x, W.pw_b[L]);                                                                        \
            __syncthreads();
            depthwise_slot<0, 0>(tid, n, x, a_base, W); contract_slot(N64{}, K4{}, 7, n, true);
            MWW_TC_BLOCK_END(0)
            depthwise_slot<1, 0>(tid, n, x, a_base, W); contract_slot(N64{}, K4{}, 8, n, true);
            depthwise_slot<1, 1>(tid, n, x, a_base, W); contract_slot(N64{}, K4{}, 9, n, false);
            MWW_TC_BLOCK_END(1)
            depthwise_slot<2, 0>(tid, n, x, a_base, W); contract_slot(N64{}, K4{}, 10, n, true);
            depthwise_slot<2, 1>(tid, n, x, a_base, W); contract_slot(N64{}, K4{}, 11, n, false);
            MWW_TC_BLOCK_END(2)
            depthwise_slot<3, 0>(tid, n, x, a_base, W); contract_slot(N64{}, K4{}, 12, n, true);
            depthwise_slot<3, 1>(tid, n, x, a_base, W); contract_slot(N64{}, K4{}, 13, n, false);
            MWW_TC_BLOCK_END(3)
#undef MWW_TC_BLOCK_END
            cp_wait<0>();
            // ---- head: 17-row window over the last block's outputs, dense(1), sigmoid ----
            {
                // thread -> (channel c = tid % 64, 32-step segment tid / 64): 17 taps in registers, X values reused along time; the
                // per-channel partial sums go through the idle operand buffers as [128 steps][pitch 65] (conflict-free both ways: lanes
                // are channels on the way in, steps on the way out), then one thread per step adds its 64
                float *part = reinterpret_cast<float *>(a_base);
                constexpr int kPp = 65;
                static_assert(128 * kPp * 4 <= 32768 + 2 * kBSlotBytes, "partial sums fit the A slot + B buffers");
                const int c = tid & 63, t0 = 32 * (tid >> 6);
                if (t0 < n) {
                    float w[17];
#pragma unroll
                    for (int r = 0; r < 17; ++r) w[r] = W.head_w[r * 64 + c];
                    const float *xc = x + c * kLdx + t0;
#pragma unroll 1
                    for (int tb = 0; tb < 32; tb += 8) {
                        float acc[8];
#pragma unroll
                        for (int i = 0; i < 8; ++i) acc[i] = 0.f;
#pragma unroll
                        for (int i = 0; i < 8 + 16; ++i) {
                            const float xv = xc[tb + i];
#pragma unroll
                            for (int tt = 0; tt < 8; ++tt) {
                                const int r = i - tt;
                                if (r >= 0 && r < 17) acc[tt] = fmaf(w[r], xv, acc[tt]);
                            }
                        }
#pragma unroll
                        for (int i = 0; i < 8; ++i) part[(t0 + tb + i) * kPp + c] = acc[i];
                    }
                }
                __syncthreads();
                if (tid < n) {
                    float acc = 0.f;
#pragma unroll 8
                    for (int cc = 0; cc < 64; ++cc) acc += part[tid * kPp + cc];
                    probs[s * probs_stream_stride + step0 + tid] = nn_sigmoid(acc + W.head_b[0]);
                }
            }
            x_to_ring<4>(tid, x, my_state, n);
            __syncthreads();                                        // X (and the feature alias) are rewritten by the next chunk
        }
        // ---- per call: new first-conv ring = the two rows before the first unconsumed one; new pending rows ----
        {
            const int consumed = 3 * n_steps;
            float ring_new = 0.f, pend_new = 0.f;
            if (tid < 80) {
                const int r = tid / kNumChannels, f = tid - r * kNumChannels;
                auto vrow = [&](int vr) -> float {                 // any virtual row of the call, from global memory
                    if (vr < 0) return my_state[(2 + vr) * kNumChannels + f];
                    if (vr < n_pend) return my_pend[vr * kNumChannels + f];
                    return (float)my_rows[(long long)(vr - n_pend) * kNumChannels + f] * kFeatureScale;
                };
                ring_new = vrow(consumed - 2 + r);
                pend_new = consumed + r < n_virtual ? vrow(consumed + r) : 0.f;
            }
            __syncthreads();
            if (tid < 80) { my_state[tid] = ring_new; my_pend[tid] = pend_new; }
            __syncthreads();                                        // `small` is reloaded for the next stream
        }
    }
}

// ---- host side -------------------------------------------------------------------------------------------------------

// 3xTF32 split and slot layout of one [K][N] weight matrix (the container's layout: input-major): slots of 32 K-values,
// each [N rows][128 B] swizzled, hi plane then lo plane
void build_tc_weights(const float *w0 /* [200][32] */, const float *const pw[4] /* [cin][64] */, std::vector<unsigned char> *blob, size_t offsets[5]) {
    blob->clear();
    std::vector<unsigned char> part;
    auto add = [&](size_t *off) {
        while (blob->size() % 256) blob->push_back(0);
        *off = blob->size();
        blob->insert(blob->end(), part.begin(), part.end());
    };
    tc_layout(w0, 200, 32, &part);
    add(&offsets[0]);
    for (int i = 0; i < 4; ++i) {
        tc_layout(pw[i], i == 0 ? 32 : 64, 64, &part);
        add(&offsets[1 + i]);
    }
}

cudaError_t launch_nn_f32_tc(const NnWeightsF32 &W, const TcWeights &TW, float *state, float *pend, int n_pend, const uint16_t *rows,
                             long long rows_stream_stride, int n_rows, float *probs, long long probs_stream_stride, int n_streams, int sm_count,
                             cudaStream_t st) {
    if (n_streams <= 0) return cudaSuccess;
    static bool done[64] = {};
    if (first_launch_on_this_device(done)) {
        cudaError_t e = cudaFuncSetAttribute(nn_f32_clip_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kTcSmemBytes);
        if (e != cudaSuccess) return e;
    }
    const int grid = n_streams < 2 * sm_count ? n_streams : 2 * sm_count;
    nn_f32_clip_tc_kernel<<<grid, kTcThreads, kTcSmemBytes, st>>>(W, TW, state, pend, n_pend, rows, rows_stream_stride, n_rows, probs,
                                                                  probs_stream_stride, n_streams);
    return cudaGetLastError();
}

}  // namespace mww
