// Host build of the frontend's branch-free scalar functions (mww_frontend_dev.cuh) next to the branching forms they
// replaced, kept here verbatim as the reference.  Each entry point returns the first input where the two disagree, or -1.
#include <stdint.h>

#include "../../microwakeword_b200/csrc/mww_frontend_dev.cuh"

using namespace mww;

namespace {

HostTables g_tables;
bool g_ready = false;
const HostTables &tables() {
    if (!g_ready) { build_host_tables(&g_tables); g_ready = true; }
    return g_tables;
}

int32_t wide_dynamic_function_branching(uint32_t x, const int16_t *lut) {
    if (x <= 2) return lut[x];
    const int interval = msb32(x);
    const int16_t *p = lut + 4 * interval - 6;
    const int32_t frac = (int32_t)(((interval < 11) ? (x << (11 - interval)) : (x >> (interval - 11))) & 0x3FF);
    int32_t r = ((int32_t)p[2] * frac) >> 5;
    r += (int32_t)((uint32_t)(int32_t)p[1] << 5);
    r *= frac;
    r = (r + (1 << 14)) >> 15;
    r += p[0];
    return (int32_t)(int16_t)r;
}

uint32_t pcan_shrink_branching(uint32_t x) {
    if (x < (2u << 12)) return (x * x) >> 20;
    return (x >> 6) - 64u;
}

uint32_t log_scale_branching(uint32_t x, const uint16_t *lut) {
    const uint32_t integer = (uint32_t)msb32(x) - 1;
    int32_t frac = (int32_t)(x - (1u << integer));
    if (integer < 16) frac <<= (16 - integer); else frac >>= (integer - 16);
    const uint32_t seg = (uint32_t)frac >> 9;
    const int32_t c0 = lut[seg], c1 = lut[seg + 1];
    const int32_t rel = ((c1 - c0) * (frac - (int32_t)(seg << 9))) >> 16;
    const uint32_t log2v = (integer << 16) + (uint32_t)(frac + c0 + rel);
    const uint32_t loge = (uint32_t)((45426ull * log2v + 32768u) >> 16);
    return ((loge << kLogScaleShift) + 32768u) >> 16;
}

uint16_t k2_output_branching(uint32_t v, uint32_t est, const int16_t *gain_lut, const uint16_t *log_lut) {
    const uint32_t scaled = v << kSmoothingBits;
    const uint32_t e = est > scaled ? scaled : est;
    const uint32_t fl = (uint32_t)(((uint64_t)v * kMinSignalRemaining) >> kNoiseBits);
    const uint32_t sub = (scaled - e) >> kSmoothingBits;
    uint32_t sig = sub > fl ? sub : fl;
    const uint32_t gain = (uint32_t)wide_dynamic_function_branching(est, gain_lut);
    const uint32_t snr = (uint32_t)(((uint64_t)sig * gain) >> kPcanSnrShift);
    sig = pcan_shrink_branching(snr);
    sig <<= kLogCorrectionBits;
    sig = sig > 1 ? log_scale_branching(sig, log_lut) : 0;
    return (uint16_t)(sig < 0xFFFFu ? sig : 0xFFFFu);
}

}  // namespace

extern "C" {

// every uint32 x in [lo, hi]: wide_dynamic_function and pcan_shrink
long long emul_forms_wdf_pcan_mismatch(uint32_t lo, uint32_t hi) {
    const int16_t *g = tables().gain_lut;
    for (uint64_t x = lo; x <= hi; ++x) {
        if (wide_dynamic_function((uint32_t)x, g) != wide_dynamic_function_branching((uint32_t)x, g)) return (long long)x;
        if (pcan_shrink((uint32_t)x) != pcan_shrink_branching((uint32_t)x)) return (long long)x;
    }
    return -1;
}

// every x in [lo, hi], lo >= 2 (the caller forms log_scale only for x > 1)
long long emul_forms_log_scale_range_mismatch(uint32_t lo, uint32_t hi) {
    const uint16_t *g = tables().log_lut;
    for (uint64_t x = lo; x <= hi; ++x)
        if (log_scale((uint32_t)x, g) != log_scale_branching((uint32_t)x, g)) return (long long)x;
    return -1;
}

// the listed x (each >= 2): index of the first mismatch
long long emul_forms_log_scale_list_mismatch(const uint32_t *x, long long n) {
    const uint16_t *g = tables().log_lut;
    for (long long i = 0; i < n; ++i)
        if (log_scale(x[i], g) != log_scale_branching(x[i], g)) return i;
    return -1;
}

// whole per-(frame, channel) output on listed (v, est) pairs
long long emul_forms_k2_output_mismatch(const uint32_t *v, const uint32_t *est, long long n) {
    const HostTables &t = tables();
    for (long long i = 0; i < n; ++i)
        if (k2_output(v[i], est[i], t.gain_lut, t.log_lut) != k2_output_branching(v[i], est[i], t.gain_lut, t.log_lut)) return i;
    return -1;
}

// windowing: mulhi_s32(s << 16, w << 4) and mulhi_s32(s's high half, w << 4) against (s * w) >> 12, every int16 s and
// every Q12 coefficient 0..4096; returns (s + 32768) * 4097 + w of the first mismatch
long long emul_forms_window_mismatch() {
    for (int32_t s = -32768; s <= 32767; ++s) {
        // s as the low and as the high sample of a packed word whose other half is not zero
        const uint32_t lo_word = 0x5A5A0000u | ((uint32_t)s & 0xFFFFu), hi_word = ((uint32_t)s << 16) | 0xA5A5u;
        for (int32_t w = 0; w <= 4096; ++w) {
            const int32_t want = (s * w) >> 12;
            if (mulhi_s32((int32_t)(lo_word << 16), w << 4) != want || mulhi_s32((int32_t)(hi_word & 0xFFFF0000u), w << 4) != want)
                return (long long)(s + 32768) * 4097 + w;
        }
    }
    return -1;
}

}  // extern "C"
