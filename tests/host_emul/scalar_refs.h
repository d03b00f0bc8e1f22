// Reference forms of the frontend's scalar functions (mww_frontend_dev.cuh, mww_common.h): the branching forms the kernels
// used before their branch-free rewrites, the library's square-root rule and the reference's float -> int16 conversion.
// Shared by the host test (emul_scalar_forms.cc) and the device harness (device_forms.cu), which compile them as host and
// as device code.  Portable integer code only: no helper here has a device intrinsic form (the msb is found with shifts),
// so a faulty intrinsic in the product cannot make both sides of a comparison agree.
#pragma once

#include <stdint.h>

#if defined(__CUDACC__)
#define REF_HD __host__ __device__ inline
#else
#define REF_HD inline
#endif

namespace ref {

// constants of the temporal chain (mww_tables.h), restated
constexpr int kSmoothingBits = 10, kNoiseBits = 14, kPcanSnrShift = 6, kLogCorrectionBits = 3, kLogScaleShift = 6;
constexpr uint32_t kMinSignalRemaining = 819;

// 1-based index of the highest set bit, 0 for x == 0
REF_HD int msb(uint32_t x) {
    int n = 0;
    if (x >> 16) { n += 16; x >>= 16; }
    if (x >> 8) { n += 8; x >>= 8; }
    if (x >> 4) { n += 4; x >>= 4; }
    if (x >> 2) { n += 2; x >>= 2; }
    if (x >> 1) { n += 1; x >>= 1; }
    return n + (int)x;
}
REF_HD int clz(uint32_t x) { return 32 - msb(x); }

REF_HD uint32_t shl_clamp(uint32_t x, int s) { return s >= 32 ? 0u : x << s; }

REF_HD uint32_t vmax_u16x2(uint32_t a, uint32_t b) {
    const uint32_t alo = a & 0xFFFFu, blo = b & 0xFFFFu, ahi = a >> 16, bhi = b >> 16;
    return (alo > blo ? alo : blo) | ((ahi > bhi ? ahi : bhi) << 16);
}

REF_HD int32_t mulhi(int32_t a, int32_t b) { return (int32_t)(((int64_t)a * (int64_t)b) >> 32); }

REF_HD int32_t wide_dynamic_function(uint32_t x, const int16_t *lut) {
    if (x <= 2) return lut[x];
    const int interval = msb(x);
    const int16_t *p = lut + 4 * interval - 6;
    const int32_t frac = (int32_t)(((interval < 11) ? (x << (11 - interval)) : (x >> (interval - 11))) & 0x3FF);
    int32_t r = ((int32_t)p[2] * frac) >> 5;
    r += (int32_t)((uint32_t)(int32_t)p[1] << 5);
    r *= frac;
    r = (r + (1 << 14)) >> 15;
    r += p[0];
    return (int32_t)(int16_t)r;
}

REF_HD uint32_t pcan_shrink(uint32_t x) {
    if (x < (2u << 12)) return (x * x) >> 20;
    return (x >> 6) - 64u;
}

REF_HD uint32_t log_scale(uint32_t x, const uint16_t *lut) {   // x >= 2
    const uint32_t integer = (uint32_t)msb(x) - 1;
    int32_t frac = (int32_t)(x - (1u << integer));
    if (integer < 16) frac <<= (16 - integer); else frac >>= (integer - 16);
    const uint32_t seg = (uint32_t)frac >> 9;
    const int32_t c0 = lut[seg], c1 = lut[seg + 1];
    const int32_t rel = ((c1 - c0) * (frac - (int32_t)(seg << 9))) >> 16;
    const uint32_t log2v = (integer << 16) + (uint32_t)(frac + c0 + rel);
    const uint32_t loge = (uint32_t)((45426ull * log2v + 32768u) >> 16);
    return ((loge << kLogScaleShift) + 32768u) >> 16;
}

REF_HD uint16_t k2_output(uint32_t v, uint32_t est, const int16_t *gain_lut, const uint16_t *log_lut) {
    const uint32_t scaled = v << kSmoothingBits;
    const uint32_t e = est > scaled ? scaled : est;
    const uint32_t fl = (uint32_t)(((uint64_t)v * kMinSignalRemaining) >> kNoiseBits);
    const uint32_t sub = (scaled - e) >> kSmoothingBits;
    uint32_t sig = sub > fl ? sub : fl;
    const uint32_t gain = (uint32_t)wide_dynamic_function(est, gain_lut);
    const uint32_t snr = (uint32_t)(((uint64_t)sig * gain) >> kPcanSnrShift);
    sig = pcan_shrink(snr);
    sig <<= kLogCorrectionBits;
    sig = sig > 1 ? log_scale(sig, log_lut) : 0;
    return (uint16_t)(sig < 0xFFFFu ? sig : 0xFFFFu);
}

// The library's rounded square root below 2^48: R = 0 for x = 0, otherwise the R with R^2 - R < x <= R^2 + R (round up
// iff the remainder exceeds the floor root), saturated at 0xFFFF when x < 2^32 (its 32-bit path).  Checks a claimed r.
REF_HD bool isqrt_below48_ok(uint64_t x, uint32_t r) {
    const uint64_t cap = (x >> 32) == 0 ? 0xFFFFull : 0xFFFFFFFFull;
    const uint64_t R = r;
    if (x == 0) return r == 0;
    if (R == cap) return x > cap * cap - cap;
    return R < cap && R * R - R < x && x <= R * R + R;
}

// audio_utils.to_int16 for one float32 sample, in double: NaN -> 0, else trunc(clamp(x * 32768, -32768, 32767))
REF_HD int16_t pcm16_from_f32(float x) {
    const double y = (double)x * 32768.0;
    if (y != y) return 0;
    const double c = y < -32768.0 ? -32768.0 : (y > 32767.0 ? 32767.0 : y);
    return (int16_t)(int32_t)c;
}

}  // namespace ref
