// mww_nn_tc.cu -- fp32 streaming MixedNet, clip formulation, on the Hopper warpgroup tensor cores (wgmma).
//
// Same graph and ring semantics as mww_nn_dev.cuh / mww_nn.cu (microwakeword/mixednet.py:307-386, layers/stream.py:581-595,
// one call = inference.py:109-123 for many steps); what changes is how the dense 88 % of the MACs -- the strided first conv
// (K = 200) and the four 1x1 projections -- are contracted:
//
//   * one CTA owns one stream and a chunk of up to 128 MODEL STEPS: time is the M dimension; each of the CTA's two warpgroups
//     contracts 64 of the steps (wgmma M = 64);
//   * the CUDA cores produce each contraction's A operand (im2col of the feature rows / the depthwise MixConv output) ONCE, already
//     split for 3xTF32 into a hi and a lo value.  The first conv's A goes straight into the wgmma register fragments; the depthwise
//     output goes to shared memory in the layout the tensor core reads: K cut into slots of 32 values = 128 bytes, a slot =
//     [128 steps][128 B] with the hardware's 128-byte XOR swizzle, so a warp whose lanes are 32 consecutive channels of one step
//     stores 128 contiguous bytes (no bank conflicts);
//   * the weights are split and laid out the same way once, at mww_create (build_tc_weights), and arrive by bulk copies from L2
//     completing on mbarriers: the first conv's seven slots at once at the start of a chunk, each 1x1 slot two slots ahead;
//   * both warpgroups issue wgmma.mma_async.m64nNk8.f32.tf32.tf32 with B (and the 1x1 projections' A) through shared-memory matrix
//     descriptors: per K = 8 step the three 3xTF32 products lo*hi, hi*lo, hi*hi accumulate into the same fp32 register tile
//     [64 steps x N];
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

// ---- shared memory map (bytes): 108.6 KB, TWO CTAs per SM -- a stream's layer chain is strictly serial (produce -> MMA -> epilogue ->
// next layer), so the only way to keep the SM busy is a second, independent stream.  Every 1x1 contraction is therefore fed ONE K-slot
// (32 input channels) at a time.  During the first conv the A slot and the B buffers hold its seven weight slots (56 KB) instead:
constexpr int kOffA = 0;                        // one K-slot of A: hi plane 16 KB + lo plane 16 KB
constexpr int kAPlaneBytes = 16384;
constexpr int kOffB = 32768;                    // two K-slots of B (double buffer): [N <= 64 rows][128 B] hi + lo = 16 KB each
constexpr int kBSlotBytes = 16384;
constexpr int kOffX = kOffB + 2 * kBSlotBytes;  // activations [64][kLdx]; the chunk's raw uint16 feature rows alias it during the first conv
constexpr int kOffSmall = kOffX + 64 * kLdx * 4;   // first-conv ring rows -2, -1 and the pending rows as floats [4][40]; then the same
                                                   // four rows as the call leaves them [4][40]
constexpr int kOffRing = kOffSmall + 8 * kNumChannels * 4;   // the next block's input ring, staged from the stream's state [R][C]
constexpr int kRingStageBytes = 22 * 64 * 4;                 // the largest ring: block 3's input
constexpr int kOffBar = kOffRing + kRingStageBytes;          // mbarriers "B buffer b holds its slot" [2], release counters [2],
                                                             // mbarrier "the first conv's weights are in place"
constexpr int kTcSmemBytes = kOffBar + 32;
static_assert(2 * (kTcSmemBytes + 1024) <= 232448, "two CTAs per SM");
static_assert(kOffRing % 16 == 0 && kOffBar % 8 == 0, "cp.async destinations and mbarriers are aligned");
static_assert(kFeatRows * kNumChannels * 2 <= 64 * kLdx * 4, "feature rows alias the activation buffer");
static_assert(kOffA % 1024 == 0 && kOffB % 1024 == 0, "swizzled operand slots need 1024-byte alignment");

// ---- phase clocks (tools/tc_phases.py builds with -DMWW_TC_PHASE_CLOCKS; compiled out of the product): thread 0 of each CTA adds
// the clock64() cycles since its previous edge to the counter of the phase that just ended.  Thread 0 waits at every CTA-wide barrier,
// so its timeline is the CTA's.
enum TcPhase {
    kPhStream, kPhFeatWait, kPhProduceFc, kPhProduceDw, kPhPublish, kPhMmaFc, kPhMmaPw, kPhRelease, kPhRingOut, kPhRingIn, kPhEpilogue,
    kPhHead, kPhCallEnd, kTcPhases
};
#ifdef MWW_TC_PHASE_CLOCKS
__device__ unsigned long long g_tc_phase_cycles[kTcPhases + 1];   // [kTcPhases]: streams completed
#define TC_PHASE_INIT long long tc_t = clock64()
#define TC_PHASE(p)                                                                                       \
    do {                                                                                                  \
        if (threadIdx.x == 0) {                                                                           \
            const long long tc_now = clock64();                                                           \
            atomicAdd(&g_tc_phase_cycles[p], (unsigned long long)(tc_now - tc_t));                        \
            tc_t = tc_now;                                                                                \
        }                                                                                                 \
    } while (0)
#else
#define TC_PHASE_INIT do {} while (0)
#define TC_PHASE(p) do {} while (0)
#endif

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
// D[64 x 32] (+)= A[64 x 8] B[8 x 32] with A from registers: a[e] = A[16 w + lane / 4 + 8 (e % 2)][lane % 4 + 4 (e / 2)] in warp w of the
// warpgroup (the tf32 register fragment); B from shared memory as above
__device__ __forceinline__ void mma_tf32_ra32(float (&d)[32], const uint32_t (&a)[4], uint64_t db, int accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
                 "{%16, %17, %18, %19}, %20, p, 1, 1;\n\t}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
                   "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(accumulate));
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
// a warpgroup's own barrier (ids 1, 2): its 128 threads only, the other warpgroup runs on
__device__ __forceinline__ void wg_sync(int wg) {
    if (wg == 0) asm volatile("bar.sync 1, 128;" ::: "memory");
    else asm volatile("bar.sync 2, 128;" ::: "memory");
}
// mbarrier + bulk copy of one weight slot (completes on the mbarrier with the byte count)
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *b, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *b, unsigned parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "W: mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra D;\n\tbra W;\n\tD:\n\t}" ::"r"(smem_u32(b)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_load(void *dst, const void *src, unsigned bytes, uint64_t *b) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(b)), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
                 "l"(__cvta_generic_to_global(src)), "r"(bytes), "r"(smem_u32(b))
                 : "memory");
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

// ring i (HBM layout [row][channel], oldest first) -> the staging buffer, 16-byte cp.async in a group of its own, issued one block
// ahead of its use so that the global-memory latency is spent under that block's work (no ring beyond the head's: I > 4 is a no-op)
template <int I>
__device__ __forceinline__ void stage_ring(int tid, float *stage, const float *ring_store) {
    if constexpr (I <= 4) {
        constexpr int n16 = tc_ring(I) * tc_cin(I) / 4;
        static_assert(n16 * 16 <= kRingStageBytes && kStateOff[I + 1] % 4 == 0, "ring fits the staging buffer in 16-byte pieces");
        const float *src = ring_store + kStateOff[I + 1];
        for (int e = tid; e < n16; e += kTcThreads) cp16(stage + 4 * e, src + 4 * e);
        cp_commit();
    }
}
// staged ring i -> history columns [0, R) of X
template <int I>
__device__ __forceinline__ void ring_to_x(int tid, float *x, const float *src) {
    constexpr int R = tc_ring(I), C = tc_cin(I);
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

// grid = min(streams, 2 x SMs) persistent CTAs (two per SM); 256 threads; one stream at a time, chunks of up to 128 model steps.
// Each warpgroup produces and contracts its own 64 steps of every K-slot (first conv: in its register fragments; 1x1: in its rows of the
// A slot), so between block ends the two warpgroups only meet at the weight buffers: a warpgroup waits on the mbarrier of the buffer
// that holds slot i, and the second warpgroup to finish slot i refills that buffer with slot i + 2 (a bulk copy from L2).  The
// CTA-wide barriers are left to the chunk start and the block ends, where the epilogues hand time steps across warpgroups.
__global__ void __launch_bounds__(kTcThreads, 2)
nn_f32_clip_tc_kernel(NnWeightsF32 W, TcWeights TW, float *__restrict__ state, float *__restrict__ pend, int n_pend, const uint16_t *__restrict__ rows,
                      long long rows_stream_stride, int n_rows, float *__restrict__ probs, long long probs_stream_stride, int n_streams) {
    extern __shared__ __align__(1024) unsigned char smem[];
    unsigned char *a_base = smem + kOffA, *b_base = smem + kOffB;
    float *x = reinterpret_cast<float *>(smem + kOffX);
    uint16_t *feat = reinterpret_cast<uint16_t *>(smem + kOffX);          // alias: dead before X's first write of a chunk
    float *small = reinterpret_cast<float *>(smem + kOffSmall);           // [0,80): first-conv ring rows -2, -1; [80,160): pending rows;
                                                                          // [160,240), [240,320): both as this call leaves them
    float *ring_stage = reinterpret_cast<float *>(smem + kOffRing);
    uint64_t *full = reinterpret_cast<uint64_t *>(smem + kOffBar);        // full[b]: B buffer b holds the slot it was last loaded with
    unsigned *released = reinterpret_cast<unsigned *>(smem + kOffBar + 16);   // warpgroups done with B buffer b, counted for ever
    uint64_t *fc_full = reinterpret_cast<uint64_t *>(smem + kOffBar + 24);     // the first conv's seven weight slots are in place
    const int tid = threadIdx.x, wg = tid >> 7;
    // this warpgroup's 64 rows of the A slot (8 KB, a whole number of 1024-byte swizzle atoms)
    const uint32_t a_s = (uint32_t)__cvta_generic_to_shared(a_base) + (uint32_t)wg * 64 * 128, b_s = (uint32_t)__cvta_generic_to_shared(b_base);
    float acc[32];
    TC_PHASE_INIT;

    // The 14 K-slots of a chunk, in order: first conv 0..6 (N = 32; the last holds K = 8), block 0 (one slot), blocks 1..3 (two each).
    // The first conv's seven slots (56 KB) arrive in one bulk copy at the start of a chunk and lie in the A slot and the B buffers, all
    // idle then: its A operand never touches shared memory (register fragments).  Slot i >= 7 sits in B buffer i % 2.
    auto load_slot = [&](int i) {                        // one thread; 7 <= i < 14
        // pointers picked by comparison, not by index: an indexed kernel parameter array would be copied to local memory
        const unsigned char *src = i == 7 ? TW.pw[0] : (i < 10 ? TW.pw[1] : i < 12 ? TW.pw[2] : TW.pw[3]) + (size_t)((i - 8) & 1) * kBSlotBytes;
        bulk_load(b_base + (i & 1) * kBSlotBytes, src, (unsigned)kBSlotBytes, full + (i & 1));
    };
    static_assert(kOffA == 0 && kOffB == 2 * kAPlaneBytes && 7 * 8192 <= kOffX, "the first conv's weights fit the A slot + B buffers");
    if (tid == 0) {
        mbar_init(full, 1);
        mbar_init(full + 1, 1);
        mbar_init(fc_full, 1);
        released[0] = released[1] = 0;
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    unsigned b_parity = 0;                               // bit b: the phase of full[b] this thread waits for next; bit 2: of fc_full
    // after this warpgroup's rows of slot i's A operand are in shared memory: publish them to the tensor core -> wait for the weights ->
    // contract (a warpgroup whose steps all lie beyond the chunk skips the MMAs, not the waits) -> release B buffer i % 2; the second
    // warpgroup to release it fetches slot i + 2 into it
    auto contract_slot = [&](auto n_out, auto ksteps, int i, int n, bool clears) {
        TC_PHASE(kPhProduceDw);
        asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
        wg_sync(wg);
        mbar_wait(full + (i & 1), (b_parity >> (i & 1)) & 1u);
        b_parity ^= 1u << (i & 1);
        TC_PHASE(kPhPublish);
        if (64 * wg < n)
            issue_slot<decltype(n_out)::value, decltype(ksteps)::value>(acc, a_s, b_s + (uint32_t)(i & 1) * kBSlotBytes, 8192u,
                                                                         clears);
        TC_PHASE(kPhMmaPw);
        wg_sync(wg);                                     // every warp of this warpgroup is past its MMAs: its A rows and B buffer i % 2 are free
        if ((tid & 127) == 0) {
            __threadfence_block();
            if ((atomicAdd(released + (i & 1), 1u) & 1u) && i + 2 < 14) load_slot(i + 2);
        }
        TC_PHASE(kPhRelease);
    };
    using N64 = std::integral_constant<int, 64>;
    using K4 = std::integral_constant<int, 4>;
    using K1 = std::integral_constant<int, 1>;

    const int n_virtual = n_pend + n_rows;
    const int n_steps = n_virtual / 3;
    for (long long s = blockIdx.x; s < n_streams; s += gridDim.x) {
        float *my_state = state + s * kStateFloats;
        float *my_pend = pend + s * 2 * kNumChannels;
        const uint16_t *my_rows = rows + s * rows_stream_stride;
        if (tid == 192) {
            // the NEXT stream's state and rows are read one stream from now: ask the L2 for them (bulk prefetch: no registers, nothing
            // to wait for)
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
            TC_PHASE(kPhStream);
            if (tid == 0) {
                // every thread fenced its generic-proxy use of these bytes before the barrier that ended the previous chunk
                asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(fc_full)), "r"(7 * 8192) : "memory");
                asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem)),
                             "l"(__cvta_generic_to_global(TW.fc)), "r"(7 * 8192), "r"(smem_u32(fc_full))
                             : "memory");
            }
            {
                const int n16 = (row_hi - row_lo) * (kNumChannels * 2 / 16);                               // 5 x 16 bytes per row
                const unsigned char *src = reinterpret_cast<const unsigned char *>(my_rows + (long long)row_lo * kNumChannels);
                for (int e = tid; e < n16; e += kTcThreads) cp16(reinterpret_cast<unsigned char *>(feat) + 16 * e, src + 16 * e);
                cp_commit();
            }
            stage_ring<0>(tid, ring_stage, my_state);
            if (step0 == 0 && tid < 160) {
                // the rows a call starts from, and -- read now, while the copies above are in flight -- the rows it leaves: the first-conv
                // ring = the two virtual rows before the first unconsumed one, the pending rows = the unconsumed ones
                const int r = tid / kNumChannels, f = tid - r * kNumChannels;
                if (tid < 80) {
                    auto vrow = [&](int vr) -> float {             // any virtual row of the call, from global memory
                        if (vr < 0) return my_state[(2 + vr) * kNumChannels + f];
                        if (vr < n_pend) return my_pend[vr * kNumChannels + f];
                        return (float)my_rows[(long long)(vr - n_pend) * kNumChannels + f] * kFeatureScale;
                    };
                    const int consumed = 3 * n_steps;
                    small[tid] = my_state[tid];
                    small[160 + tid] = vrow(consumed - 2 + r);
                    small[240 + tid] = consumed + r < n_virtual ? vrow(consumed + r) : 0.f;
                } else {
                    small[tid] = my_pend[tid - 80];
                }
            }
            cp_wait<0>();                                                  // the feature rows and block 0's ring are here
            __syncthreads();
            TC_PHASE(kPhFeatWait);
            // ---- first conv: K = 200 as seven K-slots accumulated in registers, A straight into the wgmma register fragment: thread ->
            // steps t = 64 wg + 16 w + lane / 4 (+ 8), columns lane % 4 (+ 4) of each K = 8 step (w: its warp in the warpgroup) ----
            TC_PHASE(kPhProduceFc);
            mbar_wait(fc_full, (b_parity >> 2) & 1u);
            b_parity ^= 4u;
            TC_PHASE(kPhPublish);
            {
                // both warpgroups contract, whatever n: a wgmma under a branch serialises the others (ptxas C7520); rows past the
                // chunk are zero and never stored
                const int lane = tid & 31, ta = 64 * wg + 16 * ((tid >> 5) & 3) + (lane >> 2);
                const uint32_t fc_s = (uint32_t)__cvta_generic_to_shared(smem);
                // element (t, k) is virtual row vr0 + 3 t + k / 40, column k % 40; counted in floats from row -2 it sits at
                // g = 40 (vr0 + 2) + 120 t + k, so no division: small holds g < 160, the call's rows start at g = 40 (n_pend + 2 + row_lo)
                const int g_ta = 40 * (vr0 + 2) + 120 * ta + (lane & 3), g_pend = 40 * (n_pend + 2), g_rows = 40 * (n_pend + 2 + row_lo);
                auto fc_slot = [&](auto ksteps, int slot) {
                    constexpr int KS = decltype(ksteps)::value;
                    uint32_t a_hi[KS][4], a_lo[KS][4];
#pragma unroll
                    for (int ks = 0; ks < KS; ++ks)
#pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            // steps 0 and 1 of a call's first chunk can touch the first-conv ring / the pending rows (virtual rows
                            // -2 .. n_pend - 1, in small); steps beyond the chunk contribute zero rows, never stored.  Both
                            // loads are made and one is selected: register fragments fed by divergent code would serialise the wgmmas
                            const int t = ta + 8 * (e & 1), g = g_ta + 960 * (e & 1) + 32 * slot + 8 * ks + 4 * (e >> 1);
                            const float from_small = small[min(g, 4 * kNumChannels - 1)];
                            const float from_rows = (float)feat[max(g - g_rows, 0)] * kFeatureScale;
                            const float v = t < n ? (g < g_pend ? from_small : from_rows) : 0.f;
                            float hi, lo;
                            split_tf32f(v, hi, lo);
                            a_hi[ks][e] = __float_as_uint(hi);
                            a_lo[ks][e] = __float_as_uint(lo);
                        }
                    const uint32_t b_hi0 = fc_s + (uint32_t)slot * 8192;
                    fence_acc(acc);
                    asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory");
#pragma unroll
                    for (int ks = 0; ks < KS; ++ks) {
                        const uint32_t b_hi = b_hi0 + (uint32_t)ks * 32, b_lo = b_hi + 4096;
                        mma_tf32_ra32(acc, a_lo[ks], desc_sw128(b_hi), !(slot == 0 && ks == 0));
                        mma_tf32_ra32(acc, a_hi[ks], desc_sw128(b_lo), 1);
                        mma_tf32_ra32(acc, a_hi[ks], desc_sw128(b_hi), 1);
                    }
                    asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory");
                    asm volatile("wgmma.wait_group.sync.aligned 0;\n" ::: "memory");
                    fence_acc(acc);
                };
#pragma unroll 1
                for (int slot = 0; slot < 6; ++slot) fc_slot(K4{}, slot);
                fc_slot(K1{}, 6);                                          // slot 6 only has the K = 8 step 192..199
            }
            TC_PHASE(kPhMmaFc);
            // first conv epilogue: ReLU, no bias -> X (block 0's input), its ring history in front.  The feature rows under X are dead once
            // both warpgroups are past their first-conv MMAs, and so are its weights: the B buffers take block 0's and block 1's first slot.
            __syncthreads();
            if (tid == 0) { load_slot(7); load_slot(8); }
            ring_to_x<0>(tid, x, ring_stage);
            TC_PHASE(kPhRingIn);
            epilogue<32, 4>(tid, n, acc, x, nullptr);
            __syncthreads();
            stage_ring<1>(tid, ring_stage, my_state);
            TC_PHASE(kPhEpilogue);
            // ---- four MixConv blocks: per K-slot depthwise -> contract; then ring out / next history in / epilogue / stage the ring after ----
#define MWW_TC_BLOCK_END(L)                                                                                                                 \
            x_to_ring<L>(tid, x, my_state, n);                          /* the last R columns of (history ++ outputs): the ring for later */ \
            cp_wait<0>();                                               /* ring L + 1, staged one block ago */                              \
            __syncthreads();                                                                                                                \
            TC_PHASE(kPhRingOut);                                                                                                           \
            ring_to_x<L + 1>(tid, x, ring_stage);                                                                                           \
            TC_PHASE(kPhRingIn);                                                                                                            \
            epilogue<64, tc_ring(L + 1)>(tid, n, acc, x, W.pw_b[L]);                                                                        \
            __syncthreads();                                                                                                                \
            stage_ring<L + 2>(tid, ring_stage, my_state);                                                                                   \
            TC_PHASE(kPhEpilogue);
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
            // ---- head: 17-row window over the last block's outputs, dense(1), sigmoid ----
            {
                // thread -> (channel c = tid % 64, 32-step segment tid / 64): 17 taps in registers, X values reused along time; the
                // per-channel partial sums go through the idle A slot as [128 steps][64], channel XOR (step % 32) (conflict-free both
                // ways: lanes are channels on the way in, steps on the way out), then one thread per step adds its 64 in channel order.
                // The B buffers may already be receiving the next chunk's weights.
                float *part = reinterpret_cast<float *>(a_base);
                static_assert(128 * 64 * 4 <= 2 * kAPlaneBytes, "partial sums fit the A slot");
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
                        for (int i = 0; i < 8; ++i) {
                            const int t = t0 + tb + i;
                            part[t * 64 + (c ^ (t & 31))] = acc[i];
                        }
                    }
                }
                __syncthreads();
                if (tid < n) {
                    float acc = 0.f;
#pragma unroll 8
                    for (int cc = 0; cc < 64; ++cc) acc += part[tid * 64 + (cc ^ (tid & 31))];
                    probs[s * probs_stream_stride + step0 + tid] = nn_sigmoid(acc + W.head_b[0]);
                }
            }
            x_to_ring<4>(tid, x, my_state, n);
            asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");   // the next chunk's bulk copy rewrites the A slot
            __syncthreads();                                        // X, the feature alias and the A slot are rewritten by the next chunk
            TC_PHASE(kPhHead);
        }
        // ---- per call: new first-conv ring and pending rows, read at the start of the stream (each thread writes what it read) ----
        if (tid < 80) { my_state[tid] = small[160 + tid]; my_pend[tid] = small[240 + tid]; }
        TC_PHASE(kPhCallEnd);
#ifdef MWW_TC_PHASE_CLOCKS
        if (tid == 0) atomicAdd(&g_tc_phase_cycles[kTcPhases], 1ull);
#endif
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

#ifdef MWW_TC_PHASE_CLOCKS
// phase counters of the instrumented build (tools/tc_phases.py): out[kTcPhases + 1] = cycles per phase summed over CTAs, then streams
extern "C" int mww_tc_phase_read(unsigned long long *out, int reset) {
    if (cudaDeviceSynchronize() != cudaSuccess) return 1;
    if (cudaMemcpyFromSymbol(out, mww::g_tc_phase_cycles, sizeof(mww::g_tc_phase_cycles)) != cudaSuccess) return 1;
    if (reset) {
        static const unsigned long long zero[mww::kTcPhases + 1] = {};
        if (cudaMemcpyToSymbol(mww::g_tc_phase_cycles, zero, sizeof(zero)) != cudaSuccess) return 1;
    }
    return 0;
}
#endif
