// mww_nn_i8_dev.cuh -- integer (int8-quantised) streaming MixedNet, clip formulation, per-thread phases.
//
// Executes the graph a quantised reference model runs inside tf.lite.Interpreter.invoke()
// (microwakeword/inference.py:110-121) under the conversion contract of
// microwakeword/utils.py:289-348: int8 activations (per-tensor, asymmetric), int8 weights
// (per-output-channel symmetric; per-tensor for the dense head), int32 biases, int8 ring-buffer
// state variables (:333), int8 input at scale 26/255 (:308-313), uint8 output (:338), requantised
// with TFLite's SaturatingRoundingDoublingHighMul + RoundingDivideByPOT (SURVEY.md Appendix C).
// Result is bit-exact with oracle/mixednet.c::mwwo_mixednet_step_int8.
//
// Same time-parallel shared-memory geometry as the fp32 path (mww_nn_dev.cuh); activations are
// kept as int32 words holding (q - zero_point), so a zero word is a real 0 and ring padding,
// depthwise taps and pointwise inputs need no per-use zero-point subtraction.
#pragma once

#include "mww_common.h"
#include "mww_nn_dev.cuh"

namespace mww {

struct NnWeightsI8 {
    const int8_t *w0; const int32_t *b0, *m0, *s0;              // first conv [5][40][32]
    const int8_t *dw_w[4]; const int32_t *dw_b[4], *dw_m[4], *dw_s[4];
    const int8_t *pw_w[4]; const int32_t *pw_b[4], *pw_m[4], *pw_s[4];
    const int8_t *head_w; const int8_t *lut;
    int32_t head_bias, head_mult, head_shift;
    int32_t zp[12];          // [in, c0, d1, p1, d2, p2, d3, p3, d4, p4, fc, prob]
    float in_scale;
    // tensor-core (IMMA) operands, built by mww_create from the tensors above:
    const int8_t *w0t;        // [32 n][kW0Pitch]   first-conv weights, K-contiguous (k = tap*40 + feature), zero padded
    const int8_t *pwt[4];     // [64 n][kPwPitch]   1x1 weights, K-contiguous
    const int32_t *b0f;       // [32]  bias - zp_in * sum_k w   (the MMA runs on raw int8 activations)
    const int32_t *pw_bf[4];  // [64]  bias - zp_d  * sum_k w
    // input quantisation of a uint16 feature as a table: qlut[u] = nnq_quantize(u * kFeatureScale, in_scale, zp[0]) for every
    // u (64 KB, built by mww_create / the host emulation with that very expression, so exact by construction).  nullptr: compute.
    // The table replaces a float division and conversions per feature.
    const int8_t *qlut = nullptr;
};

// zero point of the tensor buffered by ring L (0..3: block inputs, 4: head input)
MWW_HD int32_t nnq_ring_zp(const NnWeightsI8 &W, int L) { return W.zp[1 + 2 * L]; }

// MultiplyByQuantizedMultiplier (TFLite, double-rounding variant) in closed form:
//   SaturatingRoundingDoublingHighMul(a, b) = floor((a*b + 2^30) / 2^31)  for every sign of a*b: the reference's
//     nudge (2^30 | 1 - 2^30) followed by a division that truncates toward zero is exactly "round half up", i.e. an
//     ARITHMETIC 64-bit shift of (a*b + 2^30).  Its saturating case needs a == b == INT32_MIN; multipliers are >= 0.
//   RoundingDivideByPOT(x, r) = (x + half + (x < 0 ? -1 : 0)) >> r  with half = 2^(r-1)   (round half away from zero; r = 0: x)
// tests/test_host_emul.py fuzzes this against the literal SRDHM + RoundingDivideByPOT restatement of the CPU checker.
MWW_HD int32_t mbqm(int32_t x, int32_t mult, int32_t shift) {
    const int left = shift > 0 ? shift : 0, r = shift > 0 ? 0 : -shift;
    const int32_t xs = (int32_t)((uint32_t)x << left);
    const int64_t ab = (int64_t)xs * (int64_t)mult + (1ll << 30);
    const int64_t p = ab >> 31;                               // |p| <= 2^31: keep 64 bits so p + half cannot wrap
    const int64_t half = (int64_t)((1u << r) >> 1);
    const int64_t fix = (p < 0 && r) ? -1 : 0;
    return (int32_t)((p + half + fix) >> r);
}
// requantise an accumulator; returns (q_out - zp_out) so it can be stored pre-subtracted
MWW_HD int32_t requant_rel(int32_t acc, int32_t mult, int32_t shift, int32_t zp_out, bool relu) {
    int32_t y = mbqm(acc, mult, shift) + zp_out;
    const int32_t lo = relu ? zp_out : -128;
    y = y < lo ? lo : y;
    y = y > 127 ? 127 : y;
    return y - zp_out;
}

struct NnInputI8 {
    const int8_t *ring0;      // [2][40] raw int8
    const int8_t *pend;       // [2][40]
    int n_pend;
    const void *rows;
    int n_rows;
    int row_type;             // 0 uint16, 1 float32, 2 int8
};

// Model.quantize_input_data (inference.py:127-147): float divide, add zero point, astype(int8)
MWW_HD int32_t nnq_quantize(float x, float scale, int32_t zp) { return (int32_t)(int8_t)(int32_t)(x / scale + (float)zp); }

// virtual feature row element as (q - zp_in)
MWW_HD int32_t nnq_virtual_row(const NnInputI8 &in, const NnWeightsI8 &W, int vr, int f) {
    int32_t q;
    if (vr < 0) q = in.ring0[(2 + vr) * kNumChannels + f];
    else if (vr < in.n_pend) q = in.pend[vr * kNumChannels + f];
    else {
        const long long e = (long long)(vr - in.n_pend) * kNumChannels + f;
        if (in.row_type == 2) q = static_cast<const int8_t *>(in.rows)[e];
        else {
            if (in.row_type == 0 && W.qlut) q = W.qlut[static_cast<const uint16_t *>(in.rows)[e]];
            else {
                const float x = in.row_type == 1 ? static_cast<const float *>(in.rows)[e]
                                                 : (float)static_cast<const uint16_t *>(in.rows)[e] * kFeatureScale;
                q = nnq_quantize(x, W.in_scale, W.zp[0]);
            }
        }
    }
    return q - W.zp[0];
}

template <int L>
MWW_HD void nnq_load_state_l(int tid, int32_t *sm, const int8_t *state, const NnWeightsI8 &W) {
    constexpr NnLayerGeom g = kGeom[L];
    const int8_t *src = state + kStateOff[L + 1];
    const int32_t zp = nnq_ring_zp(W, L);
    for (int e = tid; e < g.ring * g.cin; e += kNnThreads) {
        const int r = e / g.cin, c = e - r * g.cin;
        sm[g.off + c * g.ld + (g.hp - g.ring) + r] = (int32_t)src[e] - zp;
    }
}
MWW_HD void nnq_load_state(int tid, int32_t *sm, const int8_t *state, const NnWeightsI8 &W) {
    nnq_load_state_l<0>(tid, sm, state, W); nnq_load_state_l<1>(tid, sm, state, W); nnq_load_state_l<2>(tid, sm, state, W);
    nnq_load_state_l<3>(tid, sm, state, W); nnq_load_state_l<4>(tid, sm, state, W);
}

// ---- tensor-core formulation of the dense int8 layers (mma.sync.m16n8k32 s8: exact int32 accumulation) -------
// M = time step, K = input channel (or tap*40 + feature), N = output channel.  Activations enter the MMA as RAW
// int8 values packed four per word along K; sum_k (q - zp) w = sum_k q w - zp * sum_k w, and the second term is
// folded into the bias on the host (b0f / pw_bf), so results equal the reference integer kernels bit for bit.
// Fragments (PTX ISA), g = lane / 4, tig = lane % 4:
//   A (16x32, row): a0 (g, 4tig..+3)  a1 (g+8, 4tig..)  a2 (g, 16+4tig..)  a3 (g+8, 16+4tig..)
//   B (32x8,  col): b0 (k = 4tig..+3, n = g)            b1 (k = 16+4tig.., n = g)
//   C (16x8)      : c0 (g, 2tig) c1 (g, 2tig+1) c2 (g+8, 2tig) c3 (g+8, 2tig+1)
// Pitches of 80 / 240 bytes (20 / 60 words) put the 8 rows x 4 words of a fragment load on 32 distinct banks.
constexpr int kPwPitch = 80;                          // bytes per row of D8 [t][k] and of the 1x1 weights [n][k]
constexpr int kW0Pitch = 240;                         // bytes per row of the first-conv im2col A8 [t][k] and of w0t [n][k]
constexpr int kMmaRows = 48;                          // 3 m-tiles of 16 steps (kTT = 36 valid)
// byte offsets inside the int8 kernel's shared memory (after the int32 ring buffers)
constexpr int kQOffD8 = kXFloats * 4;                               // packed depthwise output
constexpr int kQOffA8 = kQOffD8 + kMmaRows * kPwPitch;              // first-conv im2col; later reused as the head's int32 partial sums
constexpr int kQA8Bytes = (kMmaRows * kW0Pitch > kDFloats * 4) ? kMmaRows * kW0Pitch : kDFloats * 4;
constexpr int kQOffW0 = kQOffA8 + kQA8Bytes;
constexpr int kQOffPw = kQOffW0 + 32 * kW0Pitch;
constexpr int kNnI8SmemBytes = kQOffPw + 4 * 64 * kPwPitch;        // 102.7 KB -> 2 CTAs / SM
static_assert(kQOffD8 % 16 == 0 && kQOffA8 % 16 == 0 && kQOffW0 % 16 == 0 && kQOffPw % 16 == 0, "int8 smem carve-up");

MWW_HD int8_t *nnq_bytes(int32_t *sm) { return reinterpret_cast<int8_t *>(sm); }
MWW_HD int32_t *nnq_head_scratch(int32_t *sm) { return reinterpret_cast<int32_t *>(nnq_bytes(sm) + kQOffA8); }

// all int8 MMA weights stay resident for the whole call (28 KB)
MWW_HD void nnq_load_weights(int tid, int32_t *sm, const NnWeightsI8 &W) {
    struct alignas(16) Vec16 { uint32_t v[4]; };      // 16-byte copies (both sides are 16-byte aligned)
    int8_t *b = nnq_bytes(sm);
    for (int e = tid; e < 32 * kW0Pitch / 16; e += kNnThreads)
        reinterpret_cast<Vec16 *>(b + kQOffW0)[e] = reinterpret_cast<const Vec16 *>(W.w0t)[e];
    for (int L = 0; L < 4; ++L)
        for (int e = tid; e < 64 * kPwPitch / 16; e += kNnThreads)
            reinterpret_cast<Vec16 *>(b + kQOffPw + L * 64 * kPwPitch)[e] = reinterpret_cast<const Vec16 *>(W.pwt[L])[e];
}

// im2col of the chunk's rows as raw int8: A8[t][tap*40 + f] = q(row 3(step0+t) + tap - 2, f)
// One thread handles 8 consecutive features of one row: a single 8 / 16 / 2 x 16-byte load (int8 / uint16 / float32
// rows), eight quantisations (Model.quantize_input_data, inference.py:127-147) and one 8-byte store per im2col copy.
// The first version walked single elements -- one dependent 2-byte load, a division and two byte stores each -- and
// stalled the kernel on those dependent loads.
struct alignas(8) NnQ8 { uint32_t lo, hi; };
MWW_HD NnQ8 nnq_row_octet(const NnInputI8 &in, const NnWeightsI8 &W, int vr, int f0) {
    if (vr < 0) return *reinterpret_cast<const NnQ8 *>(in.ring0 + (2 + vr) * kNumChannels + f0);
    if (vr < in.n_pend) return *reinterpret_cast<const NnQ8 *>(in.pend + vr * kNumChannels + f0);
    const long long e = (long long)(vr - in.n_pend) * kNumChannels + f0;
    if (in.row_type == 2) return *reinterpret_cast<const NnQ8 *>(static_cast<const int8_t *>(in.rows) + e);
    float x[8];
    if (in.row_type == 1) {
        struct alignas(16) F4 { float v[4]; };
        const F4 a = *reinterpret_cast<const F4 *>(static_cast<const float *>(in.rows) + e);
        const F4 b = *reinterpret_cast<const F4 *>(static_cast<const float *>(in.rows) + e + 4);
#pragma unroll
        for (int i = 0; i < 4; ++i) { x[i] = a.v[i]; x[4 + i] = b.v[i]; }
    } else {
        struct alignas(16) U8 { uint16_t v[8]; };
        const U8 u = *reinterpret_cast<const U8 *>(static_cast<const uint16_t *>(in.rows) + e);
        if (W.qlut) {
            uint32_t t[2] = {0u, 0u};
#pragma unroll
            for (int i = 0; i < 8; ++i) t[i >> 2] |= (uint32_t)(uint8_t)W.qlut[u.v[i]] << (8 * (i & 3));
            NnQ8 r;
            r.lo = t[0]; r.hi = t[1];
            return r;
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) x[i] = (float)u.v[i] * kFeatureScale;
    }
    uint32_t w[2] = {0u, 0u};
#pragma unroll
    for (int i = 0; i < 8; ++i) w[i >> 2] |= (uint32_t)(nnq_quantize(x[i], W.in_scale, W.zp[0]) & 0xFF) << (8 * (i & 3));
    NnQ8 r;
    r.lo = w[0]; r.hi = w[1];
    return r;
}
MWW_HD void nnq_load_features(int tid, int32_t *sm, const NnInputI8 &in, const NnWeightsI8 &W, int step0, int n) {
    int8_t *a8 = nnq_bytes(sm) + kQOffA8;
    const int n_q = 3 * n + 2, U = n + 1;
    // thread -> (8-feature group, tap phase j, u) with u fastest; chunk row q = 3u + j is tap j of step u and, for
    // j < 2, tap j + 3 of step u - 1
    for (int e = tid; e < 15 * U; e += kNnThreads) {
        const int u = e % U, jf = e / U, j = jf % 3, f0 = 8 * (jf / 3);
        const int q = 3 * u + j;
        if (q >= n_q) continue;
        const NnQ8 v = nnq_row_octet(in, W, 3 * step0 + q - 2, f0);
        if (u < kMmaRows) *reinterpret_cast<NnQ8 *>(a8 + u * kW0Pitch + j * kNumChannels + f0) = v;
        if (j + 3 < 5 && u >= 1) *reinterpret_cast<NnQ8 *>(a8 + (u - 1) * kW0Pitch + (j + 3) * kNumChannels + f0) = v;
    }
}

struct FragA8 { uint32_t r[4]; };
struct FragB8 { uint32_t r[2]; };
MWW_HD void load_frag_a8(const int8_t *base, int pitch, int k0, int t0, int lane, FragA8 &a) {
    const int g = lane >> 2, tig = lane & 3;
    const int8_t *p = base + (t0 + g) * pitch + k0 + 4 * tig;
    a.r[0] = *reinterpret_cast<const uint32_t *>(p);
    a.r[1] = *reinterpret_cast<const uint32_t *>(p + 8 * pitch);
    a.r[2] = *reinterpret_cast<const uint32_t *>(p + 16);
    a.r[3] = *reinterpret_cast<const uint32_t *>(p + 8 * pitch + 16);
}
MWW_HD void load_frag_b8(const int8_t *base, int pitch, int k0, int n0, int lane, FragB8 &b) {
    const int g = lane >> 2, tig = lane & 3;
    const int8_t *p = base + (n0 + g) * pitch + k0 + 4 * tig;
    b.r[0] = *reinterpret_cast<const uint32_t *>(p);
    b.r[1] = *reinterpret_cast<const uint32_t *>(p + 16);
}
#if defined(__CUDACC__)
MWW_D void mma_s8(int32_t (&c)[4], const FragA8 &a, const FragB8 &b) {
    asm("mma.sync.aligned.m16n8k32.row.col.s32.s8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
        : "r"(a.r[0]), "r"(a.r[1]), "r"(a.r[2]), "r"(a.r[3]), "r"(b.r[0]), "r"(b.r[1]));
}
#endif

// first conv: warps 0..5 = (m-tile, pair of 8-channel tiles), 7 k-steps of 32 (K = 200 zero padded to 224)
MWW_HD void nnq_fc_store_tile(int32_t *sm, const NnWeightsI8 &W, int t0, int n0, int lane, const int32_t (&c)[4]) {
    const int g = lane >> 2, tig = lane & 3;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int t = t0 + g + ((i & 2) ? 8 : 0);
        const int o = n0 + 2 * tig + (i & 1);
        if (t < kTT) sm[kGeom[0].off + o * kGeom[0].ld + kGeom[0].hp + t] = requant_rel(c[i] + W.b0f[o], W.m0[o], W.s0[o], W.zp[1], true);
    }
}
template <int L>
MWW_HD void nnq_pw_store_tile(int32_t *sm, const NnWeightsI8 &W, int t0, int n0, int lane, const int32_t (&c)[4]) {
    constexpr NnLayerGeom gn = kGeom[L + 1];
    const int g = lane >> 2, tig = lane & 3;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int t = t0 + g + ((i & 2) ? 8 : 0);
        const int o = n0 + 2 * tig + (i & 1);
        if (t < kTT) sm[gn.off + o * gn.ld + gn.hp + t] = requant_rel(c[i] + W.pw_bf[L][o], W.pw_m[L][o], W.pw_s[L][o], W.zp[3 + 2 * L], true);
    }
}
#if defined(__CUDACC__)
MWW_D void nnq_first_conv_mma(int tid, int32_t *sm, const NnWeightsI8 &W, int n) {     // n: steps in this chunk (m-tiles beyond it are skipped)
    const int warp = tid >> 5, lane = tid & 31;
    if (warp >= 6) return;
    const int t0 = 16 * (warp >> 1), n0 = 16 * (warp & 1);
    if (t0 >= n) return;
    const int8_t *a8 = nnq_bytes(sm) + kQOffA8, *w0 = nnq_bytes(sm) + kQOffW0;
    int32_t c[2][4] = {{0, 0, 0, 0}, {0, 0, 0, 0}};
#pragma unroll
    for (int ks = 0; ks < 7; ++ks) {
        FragA8 a;
        FragB8 b0, b1;
        load_frag_a8(a8, kW0Pitch, 32 * ks, t0, lane, a);
        load_frag_b8(w0, kW0Pitch, 32 * ks, n0, lane, b0);
        load_frag_b8(w0, kW0Pitch, 32 * ks, n0 + 8, lane, b1);
        mma_s8(c[0], a, b0);
        mma_s8(c[1], a, b1);
    }
    nnq_fc_store_tile(sm, W, t0, n0, lane, c[0]);
    nnq_fc_store_tile(sm, W, t0, n0 + 8, lane, c[1]);
}
template <int L>
MWW_D void nnq_pointwise_mma(int tid, int32_t *sm, const NnWeightsI8 &W, int n) {
    constexpr int cin = kGeom[L].cin;
    const int warp = tid >> 5, lane = tid & 31;
    const int t0 = 16 * (warp / 3), nt0 = 3 * (warp % 3), ntc = (warp % 3) == 2 ? 2 : 3;
    if (t0 >= n) return;
    const int8_t *d8 = nnq_bytes(sm) + kQOffD8, *wt = nnq_bytes(sm) + kQOffPw + L * 64 * kPwPitch;
    int32_t c[3][4] = {{0, 0, 0, 0}, {0, 0, 0, 0}, {0, 0, 0, 0}};
#pragma unroll
    for (int ks = 0; ks < cin / 32; ++ks) {
        FragA8 a;
        load_frag_a8(d8, kPwPitch, 32 * ks, t0, lane, a);
        // uniform three tiles per warp (the two-tile warps recompute tile 7 into a dead accumulator): no mma.sync behind
        // a warp-dependent branch, hence no WARPSYNC / NOP wrappers (same reasoning as nn_pointwise_mma)
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            FragB8 b;
            load_frag_b8(wt, kPwPitch, 32 * ks, 8 * (nt0 + i < 8 ? nt0 + i : 7), lane, b);
            mma_s8(c[i], a, b);
        }
    }
#pragma unroll
    for (int i = 0; i < 3; ++i)
        if (i < ntc) nnq_pw_store_tile<L>(sm, W, t0, 8 * (nt0 + i), lane, c[i]);
}
#endif

template <int L, int K, int TN>
MWW_HD void nnq_depthwise_k(int c, int t0, int32_t *sm, const NnWeightsI8 &W) {
    constexpr NnLayerGeom g = kGeom[L];
    int32_t w[K];
#pragma unroll
    for (int j = 0; j < K; ++j) w[j] = W.dw_w[L][(g.kmax - K + j) * g.cin + c];
    int32_t acc[TN];
#pragma unroll
    for (int i = 0; i < TN; ++i) acc[i] = 0;
    const int32_t *x = sm + g.off + c * g.ld + (g.hp - (K - 1)) + t0;
#pragma unroll
    for (int i = 0; i < TN + K - 1; ++i) {
        const int32_t xv = x[i];
#pragma unroll
        for (int tt = 0; tt < TN; ++tt) {
            const int j = i - tt;
            if (j >= 0 && j < K) acc[tt] += w[j] * xv;
        }
    }
    const int32_t b = W.dw_b[L][c], m = W.dw_m[L][c], s = W.dw_s[L][c];
    int8_t *d8 = nnq_bytes(sm) + kQOffD8 + t0 * kPwPitch + c;
#pragma unroll
    for (int i = 0; i < TN; ++i) d8[i * kPwPitch] = (int8_t)(requant_rel(acc[i] + b, m, s, W.zp[2 + 2 * L], false) + W.zp[2 + 2 * L]);
}

template <int L>
MWW_HD void nnq_depthwise(int tid, int32_t *sm, const NnWeightsI8 &W) {
    constexpr NnLayerGeom g = kGeom[L];
    if (L == 0) {
        nnq_depthwise_k<L, g.kmax, 4>(tid & 31, 4 * (tid >> 5), sm, W);
    } else {
        if (tid >= 256) return;
        const int c = tid & 63, t0 = 9 * (tid >> 6);
        if (L == 1) { if (c < 32) nnq_depthwise_k<L, 7, 9>(c, t0, sm, W); else nnq_depthwise_k<L, 11, 9>(c, t0, sm, W); }
        else if (L == 2) { if (c < 32) nnq_depthwise_k<L, 9, 9>(c, t0, sm, W); else nnq_depthwise_k<L, 15, 9>(c, t0, sm, W); }
        else nnq_depthwise_k<L, g.kmax, 9>(c, t0, sm, W);
    }
}

MWW_HD void nnq_head_partial(int tid, int32_t *sm, const NnWeightsI8 &W) {
    constexpr NnLayerGeom g = kGeom[4];
    if (tid >= 256) return;
    const int c = tid & 63, t0 = 9 * (tid >> 6);
    int32_t w[17];
#pragma unroll
    for (int j = 0; j < 17; ++j) w[j] = W.head_w[j * 64 + c];
    int32_t acc[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) acc[i] = 0;
    const int32_t *x = sm + g.off + c * g.ld + (g.hp - 16) + t0;
#pragma unroll
    for (int i = 0; i < 9 + 16; ++i) {
        const int32_t xv = x[i];
#pragma unroll
        for (int tt = 0; tt < 9; ++tt) {
            const int j = i - tt;
            if (j >= 0 && j < 17) acc[tt] += w[j] * xv;
        }
    }
    int32_t *d = nnq_head_scratch(sm) + c * kDLd + t0;
#pragma unroll
    for (int i = 0; i < 9; ++i) d[i] = acc[i];
}

// FULLY_CONNECTED requant -> LOGISTIC LUT -> QUANTIZE to uint8 -> Model.dequantize_output_data (/255)
MWW_HD void nnq_head_finish(int tid, int32_t *sm, const NnWeightsI8 &W, int n, float *probs_out) {
    if (tid >= kTT || tid >= n) return;
    const int32_t *d = nnq_head_scratch(sm) + tid;
    int32_t acc = 0;
    for (int c = 0; c < 64; ++c) acc += d[c * kDLd];
    const int32_t logit = requant_rel(acc + W.head_bias, W.head_mult, W.head_shift, W.zp[10], false) + W.zp[10];
    const int32_t out_u8 = (int32_t)W.lut[(uint8_t)(int8_t)logit] + 128;
    probs_out[tid] = (1.0f / 255.0f) * (float)out_u8;                 // inference.py:162-170
}

template <int L>
MWW_HD void nnq_store_state_l(int tid, const int32_t *sm, int8_t *state, const NnWeightsI8 &W) {
    constexpr NnLayerGeom g = kGeom[L];
    int8_t *dst = state + kStateOff[L + 1];
    const int32_t zp = nnq_ring_zp(W, L);
    for (int e = tid; e < g.ring * g.cin; e += kNnThreads) {
        const int r = e / g.cin, c = e - r * g.cin;
        dst[e] = (int8_t)(sm[g.off + c * g.ld + (g.hp - g.ring) + r] + zp);
    }
}

struct NnTailI8 { int8_t ring_new, pend_new; };
MWW_HD void nnq_tail_read(int tid, const NnInputI8 &in, const NnWeightsI8 &W, int n_steps, int n_virtual_rows, NnTailI8 &t) {
    const int consumed = 3 * n_steps;
    t.ring_new = 0; t.pend_new = 0;
    if (tid < 2 * kNumChannels) {
        const int r = tid / kNumChannels, f = tid - r * kNumChannels;
        t.ring_new = (int8_t)(nnq_virtual_row(in, W, consumed - 2 + r, f) + W.zp[0]);
        const int vr = consumed + r;
        t.pend_new = vr < n_virtual_rows ? (int8_t)(nnq_virtual_row(in, W, vr, f) + W.zp[0]) : (int8_t)W.zp[0];
    }
}
MWW_HD void nnq_tail_write(int tid, const int32_t *sm, int8_t *state, int8_t *pend_out, const NnWeightsI8 &W, const NnTailI8 &t) {
    nnq_store_state_l<0>(tid, sm, state, W); nnq_store_state_l<1>(tid, sm, state, W); nnq_store_state_l<2>(tid, sm, state, W);
    nnq_store_state_l<3>(tid, sm, state, W); nnq_store_state_l<4>(tid, sm, state, W);
    if (tid < 2 * kNumChannels) { state[tid] = t.ring_new; pend_out[tid] = t.pend_new; }
}

// value every state byte takes after a reset: the zero point of the tensor it buffers
MWW_HD int8_t nnq_reset_value(const NnWeightsI8 &W, int e /* 0..4175 */) {
    // segment ends: first-conv ring 80, block rings 208 / 848 / 1744 / 3152, head ring 4176
    if (e < 80) return (int8_t)W.zp[0];
    if (e < 208) return (int8_t)W.zp[1];
    if (e < 848) return (int8_t)W.zp[3];
    if (e < 1744) return (int8_t)W.zp[5];
    if (e < 3152) return (int8_t)W.zp[7];
    return (int8_t)W.zp[9];
}

}  // namespace mww
