// mww_nn_mma.cuh -- tensor-core formulation of the DENSE parts of the fp32 MixedNet: the strided first
// conv (K = 200, mixednet.py:317-331) and the four 1x1 projections (mixednet.py:349-352), 88 % of the
// 24 800 MACs per model step (SURVEY.md 8d).  Depthwise convs and the 17-tap head stay on CUDA cores.
//
// Why warp-level mma (HMMA.1688.F32.TF32) and not wgmma: the contraction operands are produced by CUDA
// cores (depthwise output, im2col'ed feature planes) for ONE stream and 36 time steps at a time; a wgmma
// tile needs >= 64 rows of smem-resident, descriptor-addressed operands per warpgroup,
// and the fp32 parity budget (1e-3 on probabilities; plain TF32 measured 2.6e-3) forces the 3xTF32 split
// (hi/lo operands), which doubles the operand footprint.  With 59 KB of ring buffers per stream that leaves
// one CTA per SM and exposes the async MMA latency once per layer.  Register-fragment mma needs no extra
// shared memory, and the tensor work is ~80 m16n8k8 issues per model step -- nowhere near any tensor roofline.
// Long calls on raw uint16 rows take the 128-step wgmma kernel instead (mww_nn_tc.cu).
//
// 3xTF32: x = hi + lo with hi = x & 0xFFFFE000 (exactly representable in TF32) and lo = x - hi (exact in
// fp32, <= 13 significant bits; the hardware drops its lowest bits: relative error 2^-22 of x).
//   c += a_lo * b_hi;  c += a_hi * b_lo;  c += a_hi * b_hi     (a_lo * b_lo ~ 2^-22 is dropped)
//
// Fragment layouts of mma.m16n8k8 (PTX ISA), g = lane / 4, tig = lane % 4:
//   A (16x8, row): a0 (g, tig)  a1 (g+8, tig)  a2 (g, tig+4)  a3 (g+8, tig+4)
//   B ( 8x8, col): b0 (k = tig, n = g)         b1 (k = tig+4, n = g)
//   C (16x8)     : c0 (g, 2tig) c1 (g, 2tig+1) c2 (g+8, 2tig) c3 (g+8, 2tig+1)
// Here M = time step, K = input channel (or tap*40 + feature), N = output channel.
#pragma once

#include <string.h>

#include "mww_nn_dev.cuh"

namespace mww {

MWW_HD void split_tf32(float x, uint32_t &hi, uint32_t &lo) {
#if defined(__CUDA_ARCH__)
    const uint32_t u = __float_as_uint(x);
    hi = u & 0xFFFFE000u;
    lo = __float_as_uint(x - __uint_as_float(hi));
#else
    uint32_t u;
    memcpy(&u, &x, 4);
    hi = u & 0xFFFFE000u;
    float h, l;
    memcpy(&h, &hi, 4);
    l = x - h;
    memcpy(&lo, &l, 4);
#endif
}

struct FragA { uint32_t hi[4], lo[4]; };
struct FragB { uint32_t hi[2], lo[2]; };

// A fragment from a [k][t] array with pitch `ld` (time contiguous): rows t0+g / t0+g+8, cols k0+tig / k0+tig+4
MWW_HD void load_frag_a(const float *base, int ld, int k0, int t0, int lane, FragA &a) {
    const int g = lane >> 2, tig = lane & 3;
    const float *p = base + (k0 + tig) * ld + t0 + g;
    split_tf32(p[0], a.hi[0], a.lo[0]);
    split_tf32(p[8], a.hi[1], a.lo[1]);
    split_tf32(p[4 * ld], a.hi[2], a.lo[2]);
    split_tf32(p[4 * ld + 8], a.hi[3], a.lo[3]);
}
// A fragment from the swizzled depthwise output D (nn_d_index): k0 is a multiple of 8, so the swizzle is one constant
// per fragment half
MWW_HD void load_frag_a_d(const float *d, int k0, int t0, int lane, FragA &a) {
    const int g = lane >> 2, tig = lane & 3;
    const int s0 = ((k0 >> 2) & 7), s1 = (((k0 >> 2) + 1) & 7);
    const float *p0 = d + (k0 + tig) * kDLd, *p1 = p0 + 4 * kDLd;
    split_tf32(p0[(t0 + g) ^ s0], a.hi[0], a.lo[0]);
    split_tf32(p0[(t0 + g + 8) ^ s0], a.hi[1], a.lo[1]);
    split_tf32(p1[(t0 + g) ^ s1], a.hi[2], a.lo[2]);
    split_tf32(p1[(t0 + g + 8) ^ s1], a.hi[3], a.lo[3]);
}
// B fragment from a [k][n] array with pitch `ld` (output channel contiguous)
MWW_HD void load_frag_b(const float *base, int ld, int k0, int n0, int lane, FragB &b) {
    const int g = lane >> 2, tig = lane & 3;
    const float *p = base + (k0 + tig) * ld + n0 + g;
    split_tf32(p[0], b.hi[0], b.lo[0]);
    split_tf32(p[4 * ld], b.hi[1], b.lo[1]);
}

#if defined(__CUDACC__)
MWW_D void mma_tf32(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
    asm("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
MWW_D void mma_3xtf32(float (&c)[4], const FragA &a, const FragB &b) {
    mma_tf32(c, a.lo, b.hi);
    mma_tf32(c, a.hi, b.lo);
    mma_tf32(c, a.hi, b.hi);
}
#endif

constexpr int kWLd = kWLdDev;    // 72: pitch of the staged 1x1 weights: 72 = 8 (mod 32) -> conflict-free B fragments

// tile assignment of the 9 warps for a [36(->48) x 64] output: m-tile = warp / 3, n-tiles {0,1,2} {3,4,5} {6,7}
MWW_HD int pw_m_tile(int warp) { return warp / 3; }
MWW_HD int pw_n_first(int warp) { return 3 * (warp % 3); }
MWW_HD int pw_n_count(int warp) { return (warp % 3) == 2 ? 2 : 3; }

// epilogue of one 16x8 accumulator tile of block L's 1x1 conv: bias (folded BN), ReLU, scatter into the next
// ring buffer [o][hp + t] (columns t >= kTT do not exist)
template <int L>
MWW_HD void pw_store_tile(float *sm, const NnWeightsF32 &W, int t0, int n0, int lane, const float (&c)[4]) {
    constexpr NnLayerGeom gn = kGeom[L + 1];
    const int g = lane >> 2, tig = lane & 3;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int t = t0 + g + ((i & 2) ? 8 : 0);
        const int o = n0 + 2 * tig + (i & 1);
        if (t < kTT) {
            const float v = c[i] + W.pw_b[L][o];
            sm[gn.off + o * gn.ld + gn.hp + t] = v > 0.f ? v : 0.f;
        }
    }
}

// first conv: K = 200 = 25 k-steps of 8 (5 per tap); warp = (m-tile, k-third): k-steps [9*kt, min(25, 9*kt+9))
MWW_HD int fc_m_tile(int warp) { return warp / 3; }
MWW_HD int fc_k_begin(int warp) { return 9 * (warp % 3); }
MWW_HD int fc_k_end(int warp) { const int e = 9 * (warp % 3) + 9; return e < 25 ? e : 25; }

// A fragment of the first conv for k-step ks: tap j = ks / 5, features f0 = 8 * (ks % 5) .. +7, read from the
// de-interleaved planes (plane j % 3, time index t + j / 3)
MWW_HD void fc_load_frag_a(const float *feat, int ks, int t0, int lane, FragA &a) {
    const int j = ks / 5, f0 = 8 * (ks - 5 * j);
    load_frag_a(feat + (j % 3) * kNumChannels * kUS + j / 3, kUS, f0, t0, lane, a);
}
MWW_HD void fc_load_frag_b(const float *w0, int ks, int n0, int lane, FragB &b) {
    load_frag_b(w0, 32, 8 * ks, n0, lane, b);      // w0 is [200][32]
}
// partial sums of k-thirds 1 and 2 are parked in the (idle) D region as [kt-1][o][40]
MWW_HD void fc_store_partial(float *sm, int kt, int t0, int n0, int lane, const float (&c)[4]) {
    const int g = lane >> 2, tig = lane & 3;
    float *part = sm + kXFloats + (kt - 1) * 32 * 40;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int t = t0 + g + ((i & 2) ? 8 : 0);
        const int o = n0 + 2 * tig + (i & 1);
        if (t < kTT) part[o * 40 + t] = c[i];
    }
}
MWW_HD void fc_finish_tile(float *sm, int t0, int n0, int lane, const float (&c)[4]) {
    const int g = lane >> 2, tig = lane & 3;
    const float *part = sm + kXFloats;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int t = t0 + g + ((i & 2) ? 8 : 0);
        const int o = n0 + 2 * tig + (i & 1);
        if (t < kTT) {
            const float v = c[i] + part[o * 40 + t] + part[32 * 40 + o * 40 + t];
            sm[kGeom[0].off + o * kGeom[0].ld + kGeom[0].hp + t] = v > 0.f ? v : 0.f;
        }
    }
}

#if defined(__CUDACC__)
// ---- device phases -----------------------------------------------------------------------------

// block L's 1x1 conv on tensor cores; D[k][t] (pitch kDLd) is A, the staged weights [k][o] (pitch kWLd) are B
// `n` = model steps in this chunk: an m-tile whose 16 rows all lie beyond n is skipped by its three warps (the last chunk
// of a 100-step call has 28 steps: two m-tiles instead of three)
template <int L>
MWW_D void nn_pointwise_mma(int tid, float *sm, const NnWeightsF32 &W, int n) {
    constexpr int cin = kGeom[L].cin;
    const int warp = tid >> 5, lane = tid & 31;
    const int t0 = 16 * pw_m_tile(warp), nt0 = pw_n_first(warp), ntc = pw_n_count(warp);
    if (t0 >= n) return;
    const float *d = sm + kXFloats;
    const float *wsm = nn_pw_weight_buffer<L>(sm);
    float c[3][4];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int q = 0; q < 4; ++q) c[i][q] = 0.f;
    // Every warp issues THREE tiles' worth of MMAs: the warps that own only two n-tiles recompute tile 7 into a dead
    // accumulator.  A warp-dependent tile count put each mma.sync behind a branch the compiler cannot prove uniform, and
    // every one of them was wrapped in WARPSYNC + NOP.
    int nb[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) nb[i] = 8 * (nt0 + i < 8 ? nt0 + i : 7);
#pragma unroll 2
    for (int ks = 0; ks < cin / 8; ++ks) {
        FragA a;
        FragB b[3];
        load_frag_a_d(d, 8 * ks, t0, lane, a);
#pragma unroll
        for (int i = 0; i < 3; ++i) load_frag_b(wsm, kWLd, 8 * ks, nb[i], lane, b[i]);
        // three independent accumulator chains interleaved: a dependent HMMA never follows its predecessor directly
#pragma unroll
        for (int i = 0; i < 3; ++i) mma_tf32(c[i], a.lo, b[i].hi);
#pragma unroll
        for (int i = 0; i < 3; ++i) mma_tf32(c[i], a.hi, b[i].lo);
#pragma unroll
        for (int i = 0; i < 3; ++i) mma_tf32(c[i], a.hi, b[i].hi);
    }
#pragma unroll
    for (int i = 0; i < 3; ++i)
        if (i < ntc) pw_store_tile<L>(sm, W, t0, 8 * (nt0 + i), lane, c[i]);
}

// first conv, part a: every warp contracts its k-third for all four 8-channel tiles of its m-tile
MWW_D void nn_first_conv_mma_a(int tid, float *sm, const NnWeightsF32 &W, float (&c)[4][4], int n) {
    const int warp = tid >> 5, lane = tid & 31;
    const int t0 = 16 * fc_m_tile(warp);
    const float *feat = sm + kXFloats + kDFloats;
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int q = 0; q < 4; ++q) c[i][q] = 0.f;
    if (t0 >= n) return;
#pragma unroll 3
    for (int ks = fc_k_begin(warp); ks < fc_k_end(warp); ++ks) {
        FragA a;
        FragB b[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) fc_load_frag_b(W.w0, ks, 8 * i, lane, b[i]);     // L2-resident weights: issue first
        fc_load_frag_a(feat, ks, t0, lane, a);
#pragma unroll
        for (int i = 0; i < 4; ++i) mma_tf32(c[i], a.lo, b[i].hi);
#pragma unroll
        for (int i = 0; i < 4; ++i) mma_tf32(c[i], a.hi, b[i].lo);
#pragma unroll
        for (int i = 0; i < 4; ++i) mma_tf32(c[i], a.hi, b[i].hi);
    }
    const int kt = warp % 3;
    if (kt > 0) {
#pragma unroll
        for (int i = 0; i < 4; ++i) fc_store_partial(sm, kt, t0, 8 * i, lane, c[i]);
    }
}
// part b (after a barrier): the k-third-0 warps add the parked partial sums, ReLU, write block 0's ring buffer
MWW_D void nn_first_conv_mma_b(int tid, float *sm, const float (&c)[4][4], int n) {
    const int warp = tid >> 5, lane = tid & 31;
    if (warp % 3 != 0) return;
    const int t0 = 16 * fc_m_tile(warp);
    if (t0 >= n) return;
#pragma unroll
    for (int i = 0; i < 4; ++i) fc_finish_tile(sm, t0, 8 * i, lane, c[i]);
}
#endif

}  // namespace mww
