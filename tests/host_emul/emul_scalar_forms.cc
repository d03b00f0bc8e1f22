// Host build of the frontend's branch-free scalar functions (mww_frontend_dev.cuh) next to the branching forms they
// replaced (scalar_refs.h, shared with the device harness device_forms.cu).  Each entry point returns the first input where
// the two disagree, or -1.
#include <stdint.h>

#include "../../microwakeword_b200/csrc/mww_frontend_dev.cuh"
#include "scalar_refs.h"

using namespace mww;

namespace {

HostTables g_tables;
bool g_ready = false;
const HostTables &tables() {
    if (!g_ready) { build_host_tables(&g_tables); g_ready = true; }
    return g_tables;
}

}  // namespace

extern "C" {

// every uint32 x in [lo, hi]: wide_dynamic_function and pcan_shrink
long long emul_forms_wdf_pcan_mismatch(uint32_t lo, uint32_t hi) {
    const int16_t *g = tables().gain_lut;
    for (uint64_t x = lo; x <= hi; ++x) {
        if (wide_dynamic_function((uint32_t)x, g) != ref::wide_dynamic_function((uint32_t)x, g)) return (long long)x;
        if (pcan_shrink((uint32_t)x) != ref::pcan_shrink((uint32_t)x)) return (long long)x;
    }
    return -1;
}

// every x in [lo, hi], lo >= 2 (the caller forms log_scale only for x > 1)
long long emul_forms_log_scale_range_mismatch(uint32_t lo, uint32_t hi) {
    const uint16_t *g = tables().log_lut;
    for (uint64_t x = lo; x <= hi; ++x)
        if (log_scale((uint32_t)x, g) != ref::log_scale((uint32_t)x, g)) return (long long)x;
    return -1;
}

// the listed x (each >= 2): index of the first mismatch
long long emul_forms_log_scale_list_mismatch(const uint32_t *x, long long n) {
    const uint16_t *g = tables().log_lut;
    for (long long i = 0; i < n; ++i)
        if (log_scale(x[i], g) != ref::log_scale(x[i], g)) return i;
    return -1;
}

// whole per-(frame, channel) output on listed (v, est) pairs
long long emul_forms_k2_output_mismatch(const uint32_t *v, const uint32_t *est, long long n) {
    const HostTables &t = tables();
    for (long long i = 0; i < n; ++i)
        if (k2_output(v[i], est[i], t.gain_lut, t.log_lut) != ref::k2_output(v[i], est[i], t.gain_lut, t.log_lut)) return i;
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
