// mww_frontend_dev.cuh -- device-side micro-frontend, written as per-thread PHASE functions.
//
// Replaces the per-frame arithmetic that pymicro_features.MicroFrontend.ProcessSamples performs
// when called from microwakeword/audio/audio_utils.py:57-62 (algorithm: SURVEY.md Appendix B).
//
// Work decomposition (GPU-first, not a translation of the scalar C library):
//   * kernel K1 "spectral": every 10 ms frame is independent up to the filterbank sqrt, so a CTA of
//     256 threads processes 16 frames of one stream at a time, 16 lanes per frame:
//       P0  coalesced loads of the 18-hop audio span into shared memory (float32 audio is converted to int16 on the way)
//       P1  Q12 Hann window, packed int16x2, per-lane |max|
//       P2  input scaling + radix-4 stages 1,2 of the 256-point complex FFT on 16 register-resident
//           points per lane (bit-exact Q15 roundings of KissFFT FIXED_POINT=16)
//       P3  transpose through padded shared memory, radix-4 stages 3,4
//       P4  real-FFT post pass + |X|^2 (uint32)
//       P5  41-band triangular mel accumulation (64-bit), exact rounded integer sqrt, >> shift
//   * kernel K2 "temporal": noise-reduction IIR, PCAN gain and log scaling are the only parts that
//     carry state from frame to frame; one thread per (stream, channel) scans the frames.
//
// All functions are __host__ __device__: tests/host_emul runs them thread by thread on the CPU.
#pragma once

#include <stddef.h>

#include "mww_common.h"
#include "mww_tables.h"

#if !defined(__CUDA_ARCH__)
#include <math.h>
#endif

namespace mww {

constexpr int kFramesPerGroup = 16;
constexpr int kK1Threads = 256;
constexpr int kRowWords = 272;   // 256 + 16: two frames of one warp land in disjoint bank halves
constexpr int kGroupSamples = (kFramesPerGroup + 2) * kHop;   // 2880


// The per-lane constants of the FFT phases (window, post-pass and stage-3/4 twiddles) are kept here UNPACKED, one Int2 per
// value pair: a 64-bit load hands both halves to the multiplies with no PRMT / SHF in between, once per group and lane.
struct K1Smem {
    uint32_t A[kFramesPerGroup][kRowWords];
    uint32_t B[kFramesPerGroup][kRowWords];
    Int2 win16[240];                   // window pair p: (w[2p] << 4, w[2p+1] << 4), the scale k1_window_fft1's mulhi_s32 wants
    Int2 super_tw[128];                // real-FFT post-pass twiddles (re, im)
    Int2 lane_tw[16][15];              // stage-3 / stage-4 twiddles of lane b (re, im), see K1LaneShared
    int16_t audio[2][kGroupSamples];   // double buffered: group g+1 is prefetched (cp.async) while g is processed
    uint16_t lane_max[kFramesPerGroup][16];
    int32_t shift[kFramesPerGroup];
    int32_t fb_coef[kFbCoefWords];     // span coefficients, [slot][lane][stride] (mww_tables.h)
    int16_t gain_lut[128];             // PCAN / log tables for the temporal chain fused behind the filterbank
    uint16_t log_lut[132];
};
// 54.2 KB: above the 48 KB static limit, so the kernels take it as dynamic shared memory (opt-in per kernel and device);
// four CTAs (plus 1 KB reserved each) still fit the H100's 228 KB per SM
constexpr int kK1SmemBytes = (int)sizeof(K1Smem);
static_assert(4 * (sizeof(K1Smem) + 1024) <= 228 * 1024, "K1Smem: four CTAs per SM");
static_assert(offsetof(K1Smem, audio) % 16 == 0 && offsetof(K1Smem, lane_max) % 16 == 0, "K1Smem: 16-byte staging and lane_max rows");

// tables every K1-family kernel keeps in shared memory for its whole lifetime
MWW_HD void k1_stage_tables(int tid, K1Smem &sm, const FrontendParams &P) {
    for (int i = tid; i < kFbCoefWords; i += kK1Threads) sm.fb_coef[i] = P.fb_coef[i];
    for (int i = tid; i < 128; i += kK1Threads) sm.gain_lut[i] = P.gain_lut[i];
    for (int i = tid; i < 132; i += kK1Threads) sm.log_lut[i] = P.log_lut[i];
    for (int i = tid; i < 240; i += kK1Threads) { const uint32_t w = P.win_pairs[i]; sm.win16[i] = Int2{unpack_lo(w) << 4, unpack_hi(w) << 4}; }
    for (int i = tid; i < 128; i += kK1Threads) { const uint32_t w = P.super_tw[i]; sm.super_tw[i] = Int2{unpack_lo(w), unpack_hi(w)}; }
}

// per-thread constants that do not depend on the frame (kept in registers across groups)
struct K1Lane {
    int32_t t3r[3], t3i[3];     // stage-3 twiddles tw[4b], tw[8b], tw[12b]
    int32_t t4r[12], t4i[12];   // stage-4 twiddles tw[k'], tw[2k'], tw[3k'] for k' = 16j + b
};

// The same constants read from shared memory where they are used (15 conflict-free 64-bit LDS per group) instead of living
// in 30 registers: the clip kernel then fits 64 registers = 4 CTAs per SM (more resident warps for an issue-bound kernel).
struct K1LaneShared { const Int2 *row; };   // &sm.lane_tw[b][0]: [0..3) stage 3, [3 + 3j + q] stage 4

// ---------------------------------------------------------------------------------------------
// Q15 primitives of KissFFT FIXED_POINT=16

// C_FIXDIV(x, 4): x * (32767/4) rounded;  input must already be a valid int16 value
MWW_HD int32_t fixdiv4(int32_t x) { return (x * 8191 + 16384) >> 15; }
MWW_HD int32_t fixdiv2(int32_t x) { return (x * 16383 + 16384) >> 15; }

// C_MUL: one rounding per component
MWW_HD void cmul_q15(int32_t ar, int32_t ai, int32_t wr, int32_t wi, int32_t &mr, int32_t &mi) {
    mr = (ar * wr - ai * wi + 16384) >> 15;
    mi = (ar * wi + ai * wr + 16384) >> 15;
}

// radix-4 forward butterfly on pre-divided, pre-twiddled inputs.  Sums are left un-wrapped: every
// consumer either re-wraps (sext16 before the next multiply) or packs to int16 (implicit wrap),
// and add/sub commute with the mod-2^16 wrap, so results equal int16-storing KissFFT bit for bit.
MWW_HD void bfly4_core(int32_t &r0, int32_t &i0, int32_t &r1, int32_t &i1, int32_t &r2, int32_t &i2, int32_t &r3, int32_t &i3) {
    // scratch[0..2] = r1,r2,r3 (already multiplied by their twiddles)
    const int32_t s5r = r0 - r2, s5i = i0 - i2;
    const int32_t f0r = r0 + r2, f0i = i0 + i2;
    const int32_t s3r = r1 + r3, s3i = i1 + i3;
    const int32_t s4r = r1 - r3, s4i = i1 - i3;
    r2 = f0r - s3r; i2 = f0i - s3i;
    r0 = f0r + s3r; i0 = f0i + s3i;
    r1 = s5r + s4i; i1 = s5i - s4r;
    r3 = s5r - s4i; i3 = s5i + s4r;
}

// ---------------------------------------------------------------------------------------------
// exact integer sqrt with the library's round-half-up (remainder > root) rule

MWW_HD uint64_t sq32(uint32_t r) { return (uint64_t)r * r; }   // one 32x32->64 multiply

// Branch-free: float estimate r0 (|r0 - sqrt x| <= ~1.5e3 for x < 2^64), one Newton step in float on the EXACT
// integer residual (lands within +-1 of floor(sqrt x): the float error of the correction is < 1e-3), then two
// predicated exact fix-ups.  A third defensive pass costs a few predicated instructions and never fires.
MWW_HD uint32_t isqrt64_round(uint64_t x) {
#if defined(__CUDA_ARCH__)
    const float xf = __ull2float_rn(x);
    const float rs = rsqrtf(xf);                       // MUFU.RSQ; inf for x == 0 (handled by the final select)
    uint32_t r = __float2uint_rz(xf * rs);             // saturates at 0xFFFFFFFF
    const int64_t d = (int64_t)(x - sq32(r));
    const int64_t r1 = (int64_t)r + (int64_t)__float2int_rd(__ll2float_rn(d) * (0.5f * rs));
#else
    const float xf = (float)x;
    const float rs = x ? 1.0f / sqrtf(xf) : 0.0f;
    const float rf = xf * rs;
    uint32_t r = rf >= 4294967040.0f ? 0xFFFFFFFFu : (uint32_t)rf;
    const int64_t d = (int64_t)(x - sq32(r));
    const int64_t r1 = (int64_t)r + (int64_t)floorf((float)d * (0.5f * rs));
#endif
    r = r1 > 0xFFFFFFFFll ? 0xFFFFFFFFu : (r1 < 0 ? 0u : (uint32_t)r1);
#pragma unroll
    for (int pass = 0; pass < 2; ++pass) r -= (sq32(r) > x) ? 1u : 0u;
    uint64_t rem = x - sq32(r);
#pragma unroll
    for (int pass = 0; pass < 2; ++pass) {
        const bool up = rem > 2ull * r;
        rem -= up ? 2ull * r + 1 : 0ull;
        r += up ? 1u : 0u;
    }
    // rounding: the 32-bit fast path of the library cannot exceed 0xFFFF, the 64-bit one 0xFFFFFFFF
    const uint32_t cap = (x >> 32) == 0 ? 0xFFFFu : 0xFFFFFFFFu;
    r += (rem > r && r < cap) ? 1u : 0u;
    r = r > cap ? cap : r;
    return x == 0 ? 0u : r;
}

// The filterbank's accumulators are far below 2^48 (<= 28 bins x 12-bit weights x 31-bit energies), where the whole
// rule collapses into one IEEE double square root: x is exact in a double, s = RN(sqrt x) is within 2^-30 of the
// real root (s < 2^24), and the library's "round up iff remainder > root" is round-to-nearest of sqrt x, which never
// ties and never comes closer than 2^-27 to a half-integer (sqrt(n^2 - n) = n - 1/2 - 1/(8n) ...), so
// trunc(s + 0.5) is exact.  ~22 instructions (MUFU.RSQ64H + 10 FP64 ops) instead of ~70 integer ones; the FP64
// pipe is otherwise idle in K1.  Rejected: a branch-free variant (hand-written
// RSQ64H seed + two Newton steps + an exact integer check, all of a lane's roots in one block) -- the extra
// instructions cost more than the slow-path branch of sqrt() and the serial FP64 chains.  x >= 2^48 -- only reachable through the library's int32 view of an energy of
// exactly 2^31 -- takes the integer routine above.
MWW_HD uint32_t isqrt64_round_below48(uint64_t x) {   // x < 2^48
#if defined(__CUDA_ARCH__)
    const uint32_t r = __double2uint_rz(sqrt(__ull2double_rn(x)) + 0.5);
#else
    const uint32_t r = (uint32_t)(sqrt((double)x) + 0.5);
#endif
    const uint32_t cap = (x >> 32) == 0 ? 0xFFFFu : 0xFFFFFFFFu;      // the library's 32-bit fast path saturates at 0xFFFF
    return r > cap ? cap : r;
}
MWW_HD uint32_t isqrt64_round_fast(uint64_t x) { return (x >> 48) ? isqrt64_round(x) : isqrt64_round_below48(x); }

// ---------------------------------------------------------------------------------------------
// K1 phases

MWW_HD void k1_lane_init(int tid, const FrontendParams &P, K1Lane &L) {
    const int b = tid & 15;
    for (int j = 0; j < 3; ++j) {
        const uint32_t w = P.tw[4 * b * (j + 1)];
        L.t3r[j] = unpack_lo(w); L.t3i[j] = unpack_hi(w);
    }
    for (int j = 0; j < 4; ++j) {
        const int kp = 16 * j + b;
        for (int q = 0; q < 3; ++q) {
            const uint32_t w = P.tw[kp * (q + 1)];
            L.t4r[3 * j + q] = unpack_lo(w); L.t4i[3 * j + q] = unpack_hi(w);
        }
    }
}

MWW_HD void k1_stage_lane_twiddles(int tid, K1Smem &sm, const FrontendParams &P) {
    for (int i = tid; i < 16 * 15; i += kK1Threads) {
        const int b = i / 15, e = i - 15 * b;
        int idx;
        if (e < 3) idx = 4 * b * (e + 1);
        else { const int j = (e - 3) / 3, q = (e - 3) - 3 * j; idx = (16 * j + b) * (q + 1); }
        const uint32_t w = P.tw[idx];
        sm.lane_tw[b][e] = Int2{unpack_lo(w), unpack_hi(w)};
    }
}
MWW_HD void lane_tw3(const K1Lane &L, int q, int32_t &wr, int32_t &wi) { wr = L.t3r[q]; wi = L.t3i[q]; }
MWW_HD void lane_tw4(const K1Lane &L, int i, int32_t &wr, int32_t &wi) { wr = L.t4r[i]; wi = L.t4i[i]; }
MWW_HD void lane_tw3(const K1LaneShared &L, int q, int32_t &wr, int32_t &wi) { const Int2 w = L.row[q]; wr = w.x; wi = w.y; }
MWW_HD void lane_tw4(const K1LaneShared &L, int i, int32_t &wr, int32_t &wi) { const Int2 w = L.row[3 + i]; wr = w.x; wi = w.y; }

// ---------------------------------------------------------------------------------------------
// Caller audio comes as int16 PCM or as float32 in [-1, 1].  A float sample becomes int16 the way the reference converts
// float clips (audio_utils.py:47-48, np.clip(x * 32768, -32768, 32767).astype(np.int16)): the product in float32 (exact: a
// power-of-two scale), clamped, truncated toward zero; NaN gives 0, as numpy's cast does on x86-64.  Every kernel converts
// on load, so shared-memory staging, the window carry and all later phases only ever see int16.
MWW_HD int16_t pcm16_from_f32(float x) {
    const float y = x * 32768.0f;
    if (y != y) return 0;
    const float c = y < -32768.0f ? -32768.0f : (y > 32767.0f ? 32767.0f : y);
    return (int16_t)(int32_t)c;
}
MWW_HD int16_t pcm16(int16_t v) { return v; }
MWW_HD int16_t pcm16(float v) { return pcm16_from_f32(v); }

// P0: bring the group's audio span into shared memory.  The stream's sample sequence is
// carry[0 .. used) followed by audio[0 .. n_samples); group g needs samples [160*f0, 160*f0 + 2880).
template <typename T>
MWW_HD void k1_load_audio(int tid, K1Smem &sm, int buf, const int16_t *carry, int used, const T *audio, int n_samples, int f0) {
    const int base = kHop * f0;
    for (int i = tid; i < kGroupSamples; i += kK1Threads) {
        const int vi = base + i;
        int16_t s = 0;
        if (vi < used) s = carry[vi];
        else if (vi - used < n_samples) s = pcm16(audio[vi - used]);
        sm.audio[buf][i] = s;
    }
}

// ---- run-time hop (window_step != 10 ms; audio_utils.py:69-81 forwards step_ms to the TF op, default 20) ----
// A group holds `fpg` frames whose windows start `hop` samples apart; the whole staging area (both halves of the double
// buffer, 5 760 samples) is one span of (fpg - 1) * hop + 480 samples, loaded without prefetch.
MWW_HD int k1_hop_frames_per_group(int hop) {
    const int by_span = (2 * kGroupSamples - kWindow) / hop + 1;
    return by_span < kFramesPerGroup ? by_span : kFramesPerGroup;
}
template <typename T>
MWW_HD void k1_hop_load_audio(int tid, K1Smem &sm, const int16_t *carry, int used, const T *audio, int n_samples, int base, int span) {
    int16_t *dst = &sm.audio[0][0];
    for (int i = tid; i < span; i += kK1Threads) {
        const int vi = base + i;
        int16_t s = 0;
        if (vi < used) s = carry[vi];
        else if (vi - used < n_samples) s = pcm16(audio[vi - used]);
        dst[i] = s;
    }
}
MWW_HD int k1_hop_pair_base(int fl, int hop, int fpg) { return (hop / 2) * (fl < fpg ? fl : fpg - 1); }

// P1+P2 fused: Hann window (Q12) on the 15 sample pairs this lane owns in FFT pass 1, |max| across the
// frame's 16 lanes (half a warp), scaling to 15 significant bits, radix-4 stages 1 and 2 on the 16
// register-resident points.  PART 0 / 1 are the two halves for the host emulation (the half-warp exchange
// of lane maxima through shared memory sits between them); PART 2 is the device version.
struct K1Pass1Ctx { int32_t xr[16], xi[16]; };

// `pair_base` = word offset of the frame's first sample pair inside sm.audio[buf] (80 * slot when the 16 slots are
// consecutive frames of one stream; see k1_packed_* for the several-streams-per-CTA mapping of short calls).
template <int PART>
MWW_HD void k1_window_fft1(int tid, K1Smem &sm, int buf, int pair_base, const FrontendParams &P, K1Pass1Ctx &ctx) {
    const int fl = tid >> 4, a = tid & 15;
    const int c = (a >> 2) + 4 * (a & 3);     // complex sample index modulo 16 owned by this lane
    int32_t (&xr)[16] = ctx.xr;
    int32_t (&xi)[16] = ctx.xi;
    if (PART != 1) {
        const uint32_t *pairs = reinterpret_cast<const uint32_t *>(sm.audio[buf]) + pair_base;
        // max |v| as max(mx, -mn); a windowed value of -32768 (only reachable where the Q12 coefficient is
        // exactly 4096: samples 238..241 = pairs 119, 120 = the j == 7 column) must not win, because the
        // library's int16 negate leaves it negative.
        int32_t mx = 0, mn = 0;
#pragma unroll
        for (int b = 0; b < 16; ++b) {
            const int j = (b >> 2) + 4 * (b & 3);  // position 4*n2+n3 holds complex sample c + 16*n2 + 64*n3
            if (j == 15) { xr[b] = 0; xi[b] = 0; continue; }        // samples 480..511 are the zero padding
            const int p = c + 16 * j;
            const uint32_t sw = pairs[p];
            const Int2 cw = sm.win16[p];
            // (s * w) >> 12 as the high word of (s << 16) * (w << 4): the sample stays in its half of the packed word
            // (s << 16 is exact for int16 s, w <= 4096), and the high word is the floor, like the arithmetic shift.
            // |s| <= 32768, w <= 4096: fits int16
            const int32_t v0 = mulhi_s32((int32_t)(sw << 16), cw.x);
            const int32_t v1 = mulhi_s32((int32_t)(sw & 0xFFFF0000u), cw.y);
            xr[b] = v0; xi[b] = v1;
            if (j == 7) {
                const int32_t m0 = v0 == -32768 ? 0 : v0, m1 = v1 == -32768 ? 0 : v1;
                mx = max3i(mx, m0, m1); mn = min3i(mn, m0, m1);
            } else {
                mx = max3i(mx, v0, v1); mn = min3i(mn, v0, v1);
            }
        }
        const int32_t m = mx > -mn ? mx : -mn;
        sm.lane_max[fl][a] = (uint16_t)m;
    }
#if defined(__CUDA_ARCH__)
    if (PART == 2) __syncwarp();
#endif
    if (PART == 0) return;
    // the 16 lane maxima (each <= 32767) as packed pairs: two 128-bit loads and packed maxima
    uint32_t m2 = 0;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        uint32_t q[4];
#if defined(__CUDA_ARCH__)
        const uint4 v = reinterpret_cast<const uint4 *>(sm.lane_max[fl])[h];
        q[0] = v.x; q[1] = v.y; q[2] = v.z; q[3] = v.w;
#else
        for (int i = 0; i < 4; ++i) q[i] = (uint32_t)sm.lane_max[fl][8 * h + 2 * i] | ((uint32_t)sm.lane_max[fl][8 * h + 2 * i + 1] << 16);
#endif
        m2 = vmax_u16x2(m2, vmax_u16x2(vmax_u16x2(q[0], q[1]), vmax_u16x2(q[2], q[3])));
    }
    const uint32_t mxa = (m2 & 0xFFFFu) > (m2 >> 16) ? (m2 & 0xFFFFu) : (m2 >> 16);
    const int shift = 15 - msb32(mxa);
    if (a == 0) sm.shift[fl] = shift;
    // stage 1 (m = 1): unit twiddles; C_MUL by (32767, 0) is the identity on the pre-divided range.
    // The input scaling int16(uint16(v) << shift) is folded into C_FIXDIV's multiplier: v << shift cannot leave
    // int16 (shift comes from the maximum) except for a -32768 in the j == 7 column, which wraps like the library.
    const int32_t k4 = 8191 << shift;
#pragma unroll
    for (int g = 0; g < 4; ++g) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int b = 4 * g + q;
            const int j = (b >> 2) + 4 * (b & 3);
            if (j == 7) {
                xr[b] = fixdiv4(sext16(xr[b] << shift)); xi[b] = fixdiv4(sext16(xi[b] << shift));
            } else {
                xr[b] = (xr[b] * k4 + 16384) >> 15; xi[b] = (xi[b] * k4 + 16384) >> 15;
            }
        }
        bfly4_core(xr[4 * g], xi[4 * g], xr[4 * g + 1], xi[4 * g + 1], xr[4 * g + 2], xi[4 * g + 2], xr[4 * g + 3], xi[4 * g + 3]);
    }
    // stage 2 (m = 4): butterfly k on points k, k+4, k+8, k+12; |stage-1 sums| <= 4*8191, no wrap possible
#pragma unroll
    for (int k = 0; k < 4; ++k) {
#pragma unroll
        for (int q = 0; q < 4; ++q) { xr[k + 4 * q] = fixdiv4(xr[k + 4 * q]); xi[k + 4 * q] = fixdiv4(xi[k + 4 * q]); }
        if (k > 0) {
#pragma unroll
            for (int q = 1; q < 4; ++q) {
                int32_t mr, mi;
                cmul_q15(xr[k + 4 * q], xi[k + 4 * q], P.tw2[(k - 1) * 3 + (q - 1)][0], P.tw2[(k - 1) * 3 + (q - 1)][1], mr, mi);
                xr[k + 4 * q] = mr; xi[k + 4 * q] = mi;
            }
        }
        bfly4_core(xr[k], xi[k], xr[k + 4], xi[k + 4], xr[k + 8], xi[k + 8], xr[k + 12], xi[k + 12]);
    }
#pragma unroll
    for (int b = 0; b < 16; ++b) sm.B[fl][17 * a + b] = pack16(xr[b], xi[b]);
}

// ---- packed mapping for short calls (live mode): n_frames <= 8 frames per stream, several streams per CTA ----
// slot fl -> (stream_local = fl / fps, frame = fl % fps); every stream's span of (fps + 2) hops sits back to back in
// the (flat) audio staging area.
MWW_HD int k1_packed_streams(int fps) {
    const int by_slots = kFramesPerGroup / fps;
    const int by_smem = (2 * kGroupSamples) / ((fps + 2) * kHop);
    return by_slots < by_smem ? by_slots : by_smem;
}
template <typename T>
MWW_HD void k1_packed_load_audio(int tid, K1Smem &sm, const int16_t *carry, int used, const T *audio, long long audio_stride,
                                 int n_samples, long long s0, int n_streams, int spc, int fps) {
    const int span = (fps + 2) * kHop;
    int16_t *dst = &sm.audio[0][0];
    for (int i = tid; i < spc * span; i += kK1Threads) {
        const int sl = i / span, vi = i - sl * span;
        int16_t v = 0;
        if (s0 + sl < n_streams) {
            if (vi < used) v = carry[(s0 + sl) * kWindow + vi];
            else if (vi - used < n_samples) v = pcm16(audio[(s0 + sl) * audio_stride + (vi - used)]);
        }
        dst[i] = v;
    }
}
MWW_HD int k1_packed_pair_base(int fl, int fps) { return (fl / fps) * ((fps + 2) * (kHop / 2)) + (kHop / 2) * (fl % fps); }

// P3: transpose (lane b gathers position b of every 16-point block), FFT stages 3 and 4
template <typename LaneT>
MWW_HD void k1_fft_pass2(int tid, K1Smem &sm, const LaneT &L) {
    const int fl = tid >> 4, b = tid & 15;
    int32_t yr[16], yi[16];
#pragma unroll
    for (int a = 0; a < 16; ++a) {
        const uint32_t w = sm.B[fl][17 * a + b];
        yr[a] = unpack_lo(w); yi[a] = unpack_hi(w);
    }
    // stage 3 (m = 16, fstride 4): butterfly index k = b inside each 64-block c, points a = 4c + q
#pragma unroll
    for (int c = 0; c < 4; ++c) {
#pragma unroll
        for (int q = 0; q < 4; ++q) { yr[4 * c + q] = fixdiv4(yr[4 * c + q]); yi[4 * c + q] = fixdiv4(yi[4 * c + q]); }
#pragma unroll
        for (int q = 1; q < 4; ++q) {
            int32_t mr, mi, wr, wi;
            lane_tw3(L, q - 1, wr, wi);
            cmul_q15(yr[4 * c + q], yi[4 * c + q], wr, wi, mr, mi);
            yr[4 * c + q] = mr; yi[4 * c + q] = mi;
        }
        bfly4_core(yr[4 * c], yi[4 * c], yr[4 * c + 1], yi[4 * c + 1], yr[4 * c + 2], yi[4 * c + 2], yr[4 * c + 3], yi[4 * c + 3]);
    }
    // stage 4 (m = 64, fstride 1): butterfly index k' = 16j + b, points a = 4q + j.
    // Stage-3 sums may exceed int16; the library stored them as int16, so wrap before multiplying.
#pragma unroll
    for (int j = 0; j < 4; ++j) {
#pragma unroll
        for (int q = 0; q < 4; ++q) { yr[4 * q + j] = fixdiv4(sext16(yr[4 * q + j])); yi[4 * q + j] = fixdiv4(sext16(yi[4 * q + j])); }
#pragma unroll
        for (int q = 1; q < 4; ++q) {
            int32_t mr, mi, wr, wi;
            lane_tw4(L, 3 * j + q - 1, wr, wi);
            cmul_q15(yr[4 * q + j], yi[4 * q + j], wr, wi, mr, mi);
            yr[4 * q + j] = mr; yi[4 * q + j] = mi;
        }
        bfly4_core(yr[j], yi[j], yr[4 + j], yi[4 + j], yr[8 + j], yi[8 + j], yr[12 + j], yi[12 + j]);
    }
    // point a = 4q + j now holds bin k' + 64q = b + 16a
#pragma unroll
    for (int a = 0; a < 16; ++a) sm.A[fl][b + 16 * a] = pack16(yr[a], yi[a]);
}

// P4: split the packed complex FFT into the real spectrum and take |X|^2
MWW_HD void k1_real_energy(int tid, K1Smem &sm, const FrontendParams &P) {
    const int fl = tid >> 4, l = tid & 15;
    if (l == 0) { sm.B[fl][0] = 0; sm.B[fl][kEnergyOffset] = 0; }   // words below the first bin only ever meet zero coefficients; keep them defined
#pragma unroll
    for (int t = 0; t < 8; ++t) {
        const int k = 1 + 16 * t + l;
        const uint32_t wk = sm.A[fl][k];
        const uint32_t wn = sm.A[fl][kNcfft - k];
        const Int2 ws = sm.super_tw[k - 1];
        const int32_t pr = fixdiv2(unpack_lo(wk)), pi = fixdiv2(unpack_hi(wk));
        const int32_t nr = fixdiv2(unpack_lo(wn)), ni = fixdiv2(sext16(-unpack_hi(wn)));
        const int32_t f1r = pr + nr, f1i = pi + ni;          // |.| <= 2*16383: no wrap
        const int32_t f2r = pr - nr, f2i = pi - ni;
        int32_t tr, ti;
        cmul_q15(f2r, f2i, ws.x, ws.y, tr, ti);
        tr = sext16(tr); ti = sext16(ti);                    // C_MUL stores into int16
        // The library stores these halves as int16, but no wrap can happen: C_FIXDIV(., 2) of an int16 lies in
        // [-16383, 16383], so |f1| <= 32766, and t is an int16, so f1 +- t lies in [-65534, 65534] and its half in
        // [-32767, 32767].
        const int32_t ar = (f1r + tr) >> 1, ai = (f1i + ti) >> 1;
        const int32_t br = (f1r - tr) >> 1, bi = (ti - f1i) >> 1;
        sm.B[fl][k + kEnergyOffset] = (uint32_t)(ar * ar) + (uint32_t)(ai * ai);
        sm.B[fl][kNcfft - k + kEnergyOffset] = (uint32_t)(br * br) + (uint32_t)(bi * bi);   // for k = 128 this (later) store wins, as in the library
    }
}

// P5: mel filterbank (64-bit accumulate), rounded sqrt, undo the input scaling.  Energies and int32 coefficients come in
// two per 64-bit shared-memory load from even, conflict-free start words (mww_tables.h).
struct Pair32 { uint32_t x, y; };
MWW_HD Pair32 load_pair(const uint32_t *p) {
#if defined(__CUDA_ARCH__)
    const uint2 v = *reinterpret_cast<const uint2 *>(p);
    return Pair32{v.x, v.y};
#else
    return Pair32{p[0], p[1]};
#endif
}
MWW_HD int64_t k1_fb_accumulate(const K1Smem &sm, int fl, const FbSlot &slot, int len) {
    int64_t acc = 0;
    const uint32_t *e = &sm.B[fl][slot.word0];
    const uint32_t *cf = reinterpret_cast<const uint32_t *>(&sm.fb_coef[slot.coef_off]);
#pragma unroll
    for (int j = 0; j < len / 2; ++j) {
        const Pair32 ev = load_pair(e + 2 * j), cv = load_pair(cf + 2 * j);
        // energy widened as int32, like the library
        acc = mad_wide_s32((int32_t)ev.x, (int32_t)cv.x, acc);
        acc = mad_wide_s32((int32_t)ev.y, (int32_t)cv.y, acc);
    }
    return acc;
}
MWW_HD void k1_filterbank(int tid, K1Smem &sm, const FrontendParams &P, uint32_t *vout_frame /* [40] or nullptr */) {
    const int fl = tid >> 4, l = tid & 15;
    const int sh = sm.shift[fl];
    // An accumulator >= 2^48 needs the integer square root, and it takes a full-scale energy to make one.  The common path
    // takes the double root for every channel; if any lane of the warp met such an accumulator, the warp recomputes its
    // channels with the exact routine.  One vote per frame instead of a branch per channel.
    bool big = false;
#pragma unroll
    for (int s = 0; s < kFbSlots; ++s) {
        if (fb_len(s) == 0) continue;
        const FbSlot slot = P.fb_slots[l * kFbSlots + s];
        const uint64_t acc = (uint64_t)k1_fb_accumulate(sm, fl, slot, fb_len(s));
        big |= (acc >> 48) != 0;
        if (slot.ch >= 0 && vout_frame) vout_frame[slot.ch] = isqrt64_round_below48(acc & 0xFFFFFFFFFFFFull) >> sh;
    }
#if defined(__CUDA_ARCH__)
    big = __any_sync(0xFFFFFFFFu, big);
#endif
    if (!big || !vout_frame) return;
    for (int s = 0; s < kFbSlots; ++s) {
        if (fb_len(s) == 0) continue;
        const FbSlot slot = P.fb_slots[l * kFbSlots + s];
        if (slot.ch >= 0) vout_frame[slot.ch] = isqrt64_round_fast((uint64_t)k1_fb_accumulate(sm, fl, slot, fb_len(s))) >> sh;
    }
}

// ---------------------------------------------------------------------------------------------
// K2: per-(stream, channel) temporal chain

// Branch-free.  frac is the 10 bits below the msb (zero filled), so it is 0 for x <= 2, where the interpolation then
// returns p[0] = lut[x] by itself; p[0..2] stay inside the 125 used entries for every x (x <= 2: lut[0..4]; msb 32: lut[122..124]).
MWW_HD int32_t wide_dynamic_function(uint32_t x, const int16_t *lut) {
    const int lz = clz32(x);
    const int16_t *p = lut + (x <= 2 ? (int)x : 122 - 4 * lz);            // 4 * msb - 6
    const int32_t frac = (int32_t)((shl_clamp32(x, lz) >> 21) & 0x3FF);
    int32_t r = ((int32_t)p[2] * frac) >> 5;
    r += (int32_t)((uint32_t)(int32_t)p[1] << 5);
    r *= frac;
    r = (r + (1 << 14)) >> 15;
    r += p[0];
    return (int32_t)(int16_t)r;
}

MWW_HD uint32_t pcan_shrink(uint32_t x) {
    const uint32_t quad = (x * x) >> 20, lin = (x >> 6) - 64u;     // both formed, one selected (x * x may wrap unused)
    return x < (2u << 12) ? quad : lin;
}

MWW_HD uint32_t log_scale(uint32_t x, const uint16_t *lut) {
    // natural log of x, scaled by 2^scale_shift (SURVEY.md Appendix B step 9); defined for x >= 2.  Branch-free: frac is
    // the bits below the msb aligned to 16 bits (shifted up, zero filled, or down, truncated), which normalising x to
    // bit 31 gives in one shift.  Any x, 0 and 1 included, reads lut[0..128] only.
    const int lz = clz32(x);
    const uint32_t integer = 31u - (uint32_t)lz;
    const int32_t frac = (int32_t)(shl_clamp32(x, lz + 1) >> 16);
    const uint32_t seg = (uint32_t)frac >> 9;
    const int32_t c0 = lut[seg], c1 = lut[seg + 1];
    const int32_t rel = ((c1 - c0) * (frac - (int32_t)(seg << 9))) >> 16;
    const uint32_t log2v = (integer << 16) + (uint32_t)(frac + c0 + rel);
    const uint32_t loge = (uint32_t)((45426ull * log2v + 32768u) >> 16);
    return ((loge << kLogScaleShift) + 32768u) >> 16;
}

// The only frame-to-frame recurrence of the frontend: the noise estimate (SURVEY.md Appendix B step 7).  Returns the new
// estimate; everything else of a frame's temporal chain (k2_output) depends on it but not on other frames.
MWW_HD uint32_t k2_estimate_update(uint32_t v, uint32_t est, uint32_t smoothing) {
    const uint32_t scaled = v << kSmoothingBits;
    return (uint32_t)((((uint64_t)scaled * smoothing) + ((uint64_t)est * ((1u << kNoiseBits) - smoothing))) >> kNoiseBits);
}

// noise subtraction, PCAN and log for one channel of one frame, given the estimate AFTER this frame's update
MWW_HD uint16_t k2_output(uint32_t v, uint32_t est, const int16_t *gain_lut, const uint16_t *log_lut) {
    const uint32_t scaled = v << kSmoothingBits;
    const uint32_t e = est > scaled ? scaled : est;
    const uint32_t fl = (uint32_t)(((uint64_t)v * kMinSignalRemaining) >> kNoiseBits);
    const uint32_t sub = (scaled - e) >> kSmoothingBits;
    uint32_t sig = sub > fl ? sub : fl;
    const uint32_t gain = (uint32_t)wide_dynamic_function(est, gain_lut);
    const uint32_t snr = (uint32_t)(((uint64_t)sig * gain) >> kPcanSnrShift);
    sig = pcan_shrink(snr);
    sig <<= kLogCorrectionBits;
    const uint32_t lg = log_scale(sig, log_lut);                   // formed for every sig, kept for sig > 1
    sig = sig > 1 ? lg : 0;
    return (uint16_t)(sig < 0xFFFFu ? sig : 0xFFFFu);
}

// one frame of noise reduction + PCAN + log for one channel; `est` is the persistent noise estimate
MWW_HD uint16_t k2_channel_step(uint32_t v, uint32_t &est, uint32_t smoothing, const int16_t *gain_lut, const uint16_t *log_lut) {
    est = k2_estimate_update(v, est, smoothing);
    return k2_output(v, est, gain_lut, log_lut);
}

// ---- temporal chain fused behind the filterbank (clip kernel with one CTA per stream) -------------------------------
// After k1_filterbank has left the group's sqrt values in sm.A[frame][channel]:
//   phase 1 (threads 0..39, one per channel): the estimate recurrence over the group's frames, in order; the estimate
//            after each frame goes to sm.B[frame][channel] (the energies are dead by now), the running value stays in
//            the thread's register across groups;
//   phase 2 (all 256 threads): the 16 x 40 (frame, channel) outputs are independent given the estimates.
MWW_HD void k2_group_chain(int ch, K1Smem &sm, int n_valid, uint32_t &est) {
    const uint32_t smoothing = (ch & 1) ? kOddSmoothing : kEvenSmoothing;
    for (int f = 0; f < n_valid; ++f) {
        est = k2_estimate_update(sm.A[f][ch], est, smoothing);
        sm.B[f][ch] = est;
    }
}
MWW_HD void k2_group_outputs(int tid, K1Smem &sm, int n_valid, uint16_t *feat_group /* [n_valid][40] */) {
    for (int i = tid; i < n_valid * kNumChannels; i += kK1Threads) {
        const int f = i / kNumChannels, ch = i - f * kNumChannels;
        feat_group[i] = k2_output(sm.A[f][ch], sm.B[f][ch], sm.gain_lut, sm.log_lut);
    }
}

}  // namespace mww
