// mww_common.h -- shared macros / small integer helpers for the H100 streaming-inference kernels.
//
// Every arithmetic helper is __host__ __device__ so that tests/host_emul can execute the *same*
// phase functions the kernels run, thread by thread, on the CPU (there is no GPU in the authoring
// container).  That emulation is test infrastructure only; the product never falls back to it.
#pragma once

#include <stdint.h>

#if defined(__CUDACC__)
#define MWW_HD __host__ __device__ __forceinline__
#define MWW_D __device__ __forceinline__
#else
#define MWW_HD inline
#define MWW_D inline
#endif

namespace mww {

constexpr int kNumChannels = 40;      // mel channels (audio_utils.py:74)
constexpr int kWindow = 480;          // 30 ms @ 16 kHz (audio_utils.py:72)
constexpr int kHop = 160;             // 10 ms: pymicro_features hop (SURVEY.md 3.2)
constexpr int kFftSize = 512;
constexpr int kNcfft = 256;           // complex length of the packed real FFT
constexpr float kFeatureScale = 0.0390625f;   // inference.py:94

// leading zero bits, 32 for x == 0
MWW_HD int clz32(uint32_t x) {
#if defined(__CUDA_ARCH__)
    return __clz((int)x);
#else
    return x ? __builtin_clz(x) : 32;
#endif
}

// 1-based index of the highest set bit, 0 for x == 0
MWW_HD int msb32(uint32_t x) { return 32 - clz32(x); }

// The helpers below have a host form and a device intrinsic form.  The CPU tests (tests/test_frontend_scalar_forms.py,
// tests/test_host_emul.py) run the host forms; the device forms are covered by the GPU parity tests, which compare the
// kernels' features bit for bit with the oracle.

// x << s for 0 <= s <= 33, zero once s >= 32 (one clamped funnel shift on the device)
MWW_HD uint32_t shl_clamp32(uint32_t x, int s) {
#if defined(__CUDA_ARCH__)
    return __funnelshift_lc(0u, x, (unsigned)s);
#else
    return (uint32_t)((uint64_t)x << s);
#endif
}

// high word of the signed 32 x 32 -> 64-bit product (IMAD.HI)
MWW_HD int32_t mulhi_s32(int32_t a, int32_t b) {
#if defined(__CUDA_ARCH__)
    return __mulhi(a, b);
#else
    return (int32_t)(((int64_t)a * (int64_t)b) >> 32);
#endif
}

// per-halfword unsigned maximum of two packed uint16 pairs
MWW_HD uint32_t vmax_u16x2(uint32_t a, uint32_t b) {
#if defined(__CUDA_ARCH__)
    return __vmaxu2(a, b);
#else
    const uint32_t lo = (a & 0xFFFFu) > (b & 0xFFFFu) ? (a & 0xFFFFu) : (b & 0xFFFFu);
    const uint32_t hi = (a >> 16) > (b >> 16) ? (a >> 16) : (b >> 16);
    return lo | (hi << 16);
#endif
}

// two int32 values that one 64-bit shared-memory access moves together
struct alignas(8) Int2 { int32_t x, y; };

MWW_HD int32_t sext16(int32_t v) { return (int32_t)(int16_t)v; }

MWW_HD uint32_t pack16(int32_t lo, int32_t hi) { return ((uint32_t)lo & 0xFFFFu) | ((uint32_t)hi << 16); }
MWW_HD int32_t unpack_lo(uint32_t w) { return (int32_t)(int16_t)(w & 0xFFFFu); }
MWW_HD int32_t unpack_hi(uint32_t w) { return ((int32_t)w) >> 16; }

MWW_HD int32_t max3i(int32_t a, int32_t b, int32_t c) { const int32_t m = a > b ? a : b; return m > c ? m : c; }
MWW_HD int32_t min3i(int32_t a, int32_t b, int32_t c) { const int32_t m = a < b ? a : b; return m < c ? m : c; }

MWW_HD int64_t mad_wide_s32(int32_t a, int32_t b, int64_t c) { return (int64_t)a * (int64_t)b + c; }

}  // namespace mww
