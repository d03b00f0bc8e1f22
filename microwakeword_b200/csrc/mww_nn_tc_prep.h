// mww_nn_tc_prep.h -- the wgmma clip kernel's operand layout, shared by the kernel (mww_nn_tc.cu: the CUDA cores write the A
// operand with it, mww_create lays the weights out with it) and by the host-side test that reads the operands back the way the tensor
// core does (tests/host_emul).  No CUDA dependency.
#pragma once

#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#include <vector>

#include "mww_common.h"

namespace mww {

// Device pointers to the 3xTF32-split weights in tensor-core slot layout (laid out by mww_container.cc): K cut into slots of 32 values, a slot =
// hi plane [N rows][128 B, 128-byte swizzle] followed by the lo plane.  fc: first conv, K = 200 (7 slots), N = 32; pw[i]: 1x1 of block i.
// fc16: the first conv's weights x 0.0390625 x 2^s_fc as fp16 hi / lo operands (tc_layout_f16): K = 200 cut into 4 slots of 64, a
// slot = hi plane [32 rows][128 B] followed by the lo plane; its epilogue undoes the scale with the exact multiply fc_out = 2^-s_fc.
struct TcWeights {
    const unsigned char *fc;
    const unsigned char *pw[4];
    const unsigned char *fc16;
    float fc_out;
};

// 128-byte-swizzled K-major slot (wgmma shared-memory matrix descriptor with SWIZZLE_128B, stride byte offset 1024): rows of 128
// bytes = 32 fp32 along K; within each group of 8 rows the 16-byte chunk index is XORed with (row & 7).  Byte offset of element
// (row, kk), kk in [0, 32).
MWW_HD uint32_t sw128_off(int row, int kk) {
    return (uint32_t)row * 128u + (uint32_t)((((kk >> 2) ^ (row & 7)) << 4) + ((kk & 3) << 2));
}

// [K][N] fp32 weights -> K cut into slots of 32; per slot a hi plane [N rows][128 B swizzled] followed by the lo plane, where
// hi = the value with its low 13 mantissa bits cleared (a TF32 the tensor core reads exactly) and lo = value - hi (exact in fp32);
// positions k >= K of the last slot are zero.
inline void tc_layout(const float *w, int K, int N, std::vector<unsigned char> *out) {
    const int slots = (K + 31) / 32, plane = N * 128;
    out->assign((size_t)slots * 2 * plane, 0);
    for (int k = 0; k < K; ++k)
        for (int n = 0; n < N; ++n) {
            const float v = w[(size_t)k * N + n];
            uint32_t u;
            memcpy(&u, &v, 4);
            const uint32_t hu = u & 0xFFFFE000u;
            float hi, lo;
            memcpy(&hi, &hu, 4);
            lo = v - hi;
            unsigned char *slot = out->data() + (size_t)(k >> 5) * 2 * plane;
            memcpy(slot + sw128_off(n, k & 31), &hi, 4);
            memcpy(slot + plane + sw128_off(n, k & 31), &lo, 4);
        }
}

// ---- fp16 hi / lo operands ------------------------------------------------------------------------------------------------
// The same 128-byte rows hold 64 fp16 along K: byte offset of element (row, kk), kk in [0, 64).
MWW_HD uint32_t sw128_off_h(int row, int kk) {
    return (uint32_t)row * 128u + (uint32_t)((((kk >> 3) ^ (row & 7)) << 4) + ((kk & 7) << 1));
}

// Largest uint16 feature the frontend emits: log_scale() (mww_frontend_dev.cuh) of any 32-bit input is at most
// ((loge << 6) + 32768) >> 16 with log2 in [31, 32), i.e. 1 420 (tests/test_tc_f16.py derives it from the table).  Every
// integer up to 2048 is exact in fp16, so a feature row is an exact fp16 A operand.
constexpr int kTcMaxFeature = 1420;
// A call of at least this many model steps leaves first-conv ring and pending rows made of its own rows only: 3 x 2 - 2 >= the
// at most 2 rows pending before it.
constexpr int kTcFreshSteps = 2;

// fp16 round-to-nearest-even of |x| < 65520 (subnormals included), as bits
inline uint16_t f16_bits_rn(double x) {
    const uint16_t sign = x < 0 ? 0x8000 : 0;
    const double a = fabs(x);
    if (a < 0x1p-14) return (uint16_t)(sign | (uint16_t)nearbyint(a * 0x1p24));    // 1024 rounds up to the smallest normal's bits
    int e;
    frexp(a, &e);                                                                   // a in [2^(e-1), 2^e)
    double m = nearbyint(ldexp(a, 11 - e));                                         // 11 significant bits: [1024, 2048]
    int E = e - 1;
    if (m == 2048.0) { m = 1024.0; E += 1; }
    return (uint16_t)(sign | (uint16_t)((E + 15) << 10) | (uint16_t)(m - 1024.0));
}
inline double f16_value(uint16_t h) {
    const int E = (h >> 10) & 31, m = h & 1023;
    const double v = E == 0 ? ldexp((double)m, -24) : ldexp((double)(1024 + m), E - 25);
    return (h & 0x8000) ? -v : v;
}

// Power-of-two exponent s with max_abs * 2^s in [2^14, 2^15): the scaled values and their fp16 hi parts stay below 2^15, half of
// fp16's range, and lo = x - hi stays normal for every |x| >= max_abs * 2^-17.
inline int f16_scale_exp(double max_abs) {
    if (!(max_abs > 0)) return 0;
    int e;
    frexp(max_abs, &e);                                                             // max_abs in [2^(e-1), 2^e)
    return 15 - e;
}

// [K][N] weights times `mul` (exact in double) times 2^s -> K cut into slots of 64; per slot an fp16 hi plane [N rows][128 B
// swizzled] followed by the lo plane, hi = fp16(x), lo = fp16(x - hi); positions k >= K of the last slot are zero.
inline void tc_layout_f16(const float *w, int K, int N, double mul, int s, std::vector<unsigned char> *out) {
    const int slots = (K + 63) / 64, plane = N * 128;
    out->assign((size_t)slots * 2 * plane, 0);
    for (int k = 0; k < K; ++k)
        for (int n = 0; n < N; ++n) {
            const double x = ldexp((double)w[(size_t)k * N + n] * mul, s);
            const uint16_t hi = f16_bits_rn(x), lo = f16_bits_rn(x - f16_value(hi));
            unsigned char *slot = out->data() + (size_t)(k >> 6) * 2 * plane;
            memcpy(slot + sw128_off_h(n, k & 63), &hi, 2);
            memcpy(slot + plane + sw128_off_h(n, k & 63), &lo, 2);
        }
}

// The first conv's fp16 scheme for a model: A = u is exact, the weights w0' = w0 x 0.0390625 x 2^s_fc are an fp16 hi / lo pair
// (f16_scale_exp of the largest |w0'|).  ok = false keeps the 3xTF32 first conv: a weight that is not finite or not below 2^100, or
// an output channel whose largest |w0'| lies more than 2^17 below the tensor's largest -- there lo drops into fp16's subnormals and
// that channel keeps fewer than the 22 significant bits of a tf32 hi / lo pair.
struct TcF16Scales {
    bool ok;
    int s_fc;
};
inline TcF16Scales tc_f16_scales(const float *w0 /* [200][32] */) {
    double col[32] = {}, mx = 0;
    bool finite = true;
    for (int k = 0; k < 200; ++k)
        for (int n = 0; n < 32; ++n) {
            const double a = fabs((double)w0[k * 32 + n] * 0.0390625);
            finite = finite && a < 0x1p100;                 // false for a NaN too
            col[n] = a > col[n] ? a : col[n];
            mx = a > mx ? a : mx;
        }
    TcF16Scales r{finite, f16_scale_exp(mx)};
    for (int n = 0; n < 32; ++n)
        if (col[n] != 0 && col[n] < ldexp(mx, -17)) r.ok = false;
    return r;
}

}  // namespace mww
