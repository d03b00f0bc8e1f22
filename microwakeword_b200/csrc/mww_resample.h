// mww_resample.h -- the input-rate resampler in front of the frontend (mww_set_input_rate): filter design, polyphase table
// and the streaming index math of resample_kernel (mww_resample.cu).  CUDA-free apart from MWW_HD, so that
// tests/emul_resample.cc runs the same functions on the CPU.
//
// Definition (integers only).  For an input rate fs with L / M = 16000 / fs in lowest terms and int16 Q15 taps h[0, N):
//
//     y[n] = sat16((sum_j h[j] * x_up[n M - j] + 2^14) >> 15),   x_up = x zero-stuffed by L
//
// which is scipy.signal.upfirdn(h, x, L, M) followed by the rounding shift.  The sum is formed exactly: the taps of one
// output (one phase of the polyphase table) go into two int32 partial sums, alternate taps each, and the design checks that
// each half's sum of |h| is below 2^16, so neither partial sum can leave int32 for any int16 input; the two are added in 64
// bits.  Streams are causal: after N input samples a stream has emitted ceil(N L / M) outputs, the prefix of one upfirdn
// over everything it was given, and output n reads inputs up to floor(n M / L) only.  Each stream carries the last
// H = ceil(N / L) input samples as history.
#pragma once

#include <math.h>
#include <stdint.h>
#include <stdlib.h>

#include <vector>

#include "mww_common.h"

namespace mww {

constexpr int kResampleRates[] = {8000, 16000, 22050, 24000, 32000, 44100, 48000};
constexpr double kResampleAttenDb = 80.0;      // Kaiser design attenuation (scipy.signal.kaiserord's `ripple`)
constexpr int kResampleMaxTaps = 40000;        // the longest design (22.05 / 44.1 kHz) has 35 413

// one input rate's filter: L / M, tap count N, taps per phase T, history H (= T) and the padded row pitch of the
// phase-major table the kernel keeps in shared memory (even, half of it odd: lanes on different phases hit different banks)
struct ResamplePlan {
    int rate = 16000, L = 1, M = 1, n_taps = 0, T = 0, H = 0, pitch = 0;
    double pass_hz = 0, stop_hz = 0, beta = 0;
};

// one resample_kernel launch over a tile of streams: table [L][pitch] and history [n_streams][hist_stride] (first H used)
// in device memory, the call's n_in input samples per stream -> its n_out outputs, the first at t0 (resample_t0)
struct ResampleArgs {
    const int16_t *table = nullptr;
    int16_t *hist = nullptr;
    long long audio_stride = 0, out_stride = 0;
    int hist_stride = 0, L = 1, M = 1, T = 0, H = 0, pitch = 0, t0 = 0, n_in = 0, n_out = 0, n_streams = 0;
};

inline int resample_gcd(int a, int b) { while (b) { const int t = a % b; a = b; b = t; } return a; }

// false for a rate outside the list.  16 000 Hz: L = M = 1 and no filter (n_taps 0): no resampler runs.
inline bool resample_plan(int rate, ResamplePlan *P) {
    bool listed = false;
    for (int r : kResampleRates) listed = listed || r == rate;
    if (!listed) return false;
    ResamplePlan R;
    R.rate = rate;
    const int g = resample_gcd(16000, rate);
    R.L = 16000 / g; R.M = rate / g;
    if (rate != 16000) {
        // 8 kHz is interpolated only: transition band 0.45 .. 0.55 fs_in.  Every other rate is decimated: pass to 7 500 Hz (the
        // mel filterbank's upper band edge), stop from 8 500 Hz, so whatever folds back lands above 7 500 Hz.
        R.pass_hz = rate == 8000 ? 0.45 * rate : 7500.0;
        R.stop_hz = rate == 8000 ? 0.55 * rate : 8500.0;
        const double fs_up = (double)rate * R.L;
        const double width = (R.stop_hz - R.pass_hz) / (fs_up / 2);
        const double A = kResampleAttenDb;
        R.beta = A > 50 ? 0.1102 * (A - 8.7) : (A > 21 ? 0.5842 * pow(A - 21, 0.4) + 0.07886 * (A - 21) : 0.0);
        R.n_taps = (int)ceil((A - 7.95) / 2.285 / (M_PI * width) + 1) | 1;      // kaiserord's length, made odd (symmetric, type I)
        R.T = (R.n_taps + R.L - 1) / R.L;
        R.H = R.T;
        int half = (R.T + 1) / 2;
        if (half % 2 == 0) ++half;
        R.pitch = 2 * half;
    }
    *P = R;
    return true;
}

// modified Bessel function of the first kind, order 0 (power series; converges for the beta of any attenuation used here)
inline double resample_i0(double x) {
    double s = 1, t = 1;
    for (int k = 1; k < 200; ++k) {
        t *= (x / (2 * k)) * (x / (2 * k));
        s += t;
        if (t < s * 1e-17) break;
    }
    return s;
}

// Taps of plan P (P.n_taps of them, int16 range, held in int32): scipy.signal.firwin(N, (pass + stop) / 2,
// window=('kaiser', beta), fs=L fs) -- windowed sinc normalised to unit DC gain -- times L (the gain zero-stuffing takes
// away), times 2^15, rounded half away from zero and clamped to int16 (only 8 kHz's centre tap, exactly 1.0, is clamped:
// 32 768 becomes 32 767).  Returns false if a phase breaks the partial-sum bound (never for the listed rates).
inline bool resample_taps(const ResamplePlan &P, int32_t *out) {
    const int N = P.n_taps;
    if (N <= 0) return true;
    const double c = (P.pass_hz + P.stop_hz) / 2 / ((double)P.rate * P.L / 2);      // cutoff over the upsampled Nyquist
    const double alpha = 0.5 * (N - 1), i0b = resample_i0(P.beta);
    if (N > kResampleMaxTaps) return false;
    std::vector<double> h((size_t)N);
    double sum = 0;
    for (int i = 0; i < N; ++i) {
        const double m = i - alpha, xm = c * m;
        const double sinc = xm == 0 ? 1.0 : sin(M_PI * xm) / (M_PI * xm);
        const double r = (i - alpha) / alpha;
        h[i] = c * sinc * resample_i0(P.beta * sqrt(fmax(0.0, 1 - r * r))) / i0b;
        sum += h[i];
    }
    for (int i = 0; i < N; ++i) {
        double v = llround(h[i] / sum * P.L * 32768.0);
        v = v > 32767 ? 32767 : (v < -32768 ? -32768 : v);
        out[i] = (int32_t)v;
    }
    for (int p = 0; p < P.L; ++p) {
        long long s[2] = {0, 0};
        for (int i = 0; p + i * P.L < N; ++i) s[i & 1] += llabs(out[p + i * P.L]);
        if (s[0] >= 65536 || s[1] >= 65536) return false;
    }
    return true;
}

// phase-major table [L][pitch]: row p holds h[p], h[p + L], h[p + 2L], ... (zero past the end)
inline void resample_table(const ResamplePlan &P, const int32_t *taps, int16_t *table) {
    for (int p = 0; p < P.L; ++p)
        for (int i = 0; i < P.pitch; ++i) {
            const long long j = p + (long long)i * P.L;
            table[(size_t)p * P.pitch + i] = (int16_t)(i < P.T && j < P.n_taps ? taps[j] : 0);
        }
}

// outputs a stream has emitted after n_in input samples: ceil(n_in L / M)
MWW_HD long long resample_outputs(long long n_in, int L, int M) { return (n_in * L + M - 1) / M; }
// outputs of a call of n samples after `seen` inputs (everything before the call)
inline int resample_call_outputs(long long seen, int n, int L, int M) {
    return (int)(resample_outputs(seen + n, L, M) - resample_outputs(seen, L, M));
}
// t0 of a call after `seen` inputs: its first output n0 = ceil(seen L / M) sits at n0 M - seen L in [0, M) upsampled samples
// past the call's first input; only seen mod M matters
inline int resample_t0(long long seen, int L, int M) {
    const long long r = (seen % M) * L % M;
    return (int)((M - r) % M);
}

// Per-stream rates (mww_set_stream_rates).  The handle counts t, the 16 kHz samples every stream has been given.  A stream at
// rate r (L / M = 16000 / r) has then been given N(t) = floor(t M / L) input samples, and a call of n16 takes
// N(t + n16) - N(t) of them.  For even t, ceil(N(t) L / M) = t: write t M = N L + rho with 0 <= rho < L.  Then N L <= t M,
// and at 8 kHz (L = 2, M = 1) rho = 0 since t is even, so N L = t M; at every other rate M >= L > rho, so N L > t M - M.
// Either way (t - 1) M < N L <= t M.  So the stream's resampler has emitted exactly t outputs, and a call of even n16 gives
// every stream n16 of them, whatever its rate.
MWW_HD long long resample_inputs(long long t16, int L, int M) { return t16 * M / L; }

// the largest history H of any listed rate: the row length of the per-stream-rate history
inline int resample_max_history() {
    int h = 0;
    for (int r : kResampleRates) {
        ResamplePlan P;
        resample_plan(r, &P);
        h = P.H > h ? P.H : h;
    }
    return h;
}

// Which rows stream index s of a resample_kernel launch reads and writes.  TileRows: the tile's streams in order (a handle
// with one input rate).  MemberRows: the members of one rate in the tile, ids[0, n) sorted global ids (per-stream rates):
// input and output rows ids[s] - first of the tile, history row ids[s] of the handle.  A plan without taps (16 kHz) is the
// identity there: output q = pcm16(input q), no history.  MixedRows (below): MemberRows with a sample format per stream.
struct TileRows {
    static constexpr bool kGathered = false, kMixed = false;
    MWW_HD int io(int s) const { return s; }
    MWW_HD int hist(int s) const { return s; }
};
struct MemberRows {
    static constexpr bool kGathered = true, kMixed = false;
    const int32_t *ids; int first;
    MWW_HD int io(int s) const { return ids[s] - first; }
    MWW_HD int hist(int s) const { return ids[s]; }
};

// Per-stream sample formats (mww_set_stream_formats): the codes of include/mww.h, and the bytes one sample of each takes.
// A row of mixed audio (the _mixed entry points) is bytes: row s holds D_s samples of stream s's own format, with the row
// pitch in bytes; Mixed8 is one such byte, the sample type the call bodies of mww_capi.cu carry for these rows.
constexpr int kFormatS16 = 0, kFormatUlaw = 1, kFormatAlaw = 2, kFormatF32 = 3, kNumFormats = 4;
MWW_HD int format_bytes(int f) { return f == kFormatF32 ? 4 : (f == kFormatS16 ? 2 : 1); }
struct Mixed8 { uint8_t v; };
// MemberRows whose rows are bytes in each member's own format, fmt [n_streams] by global id (the resampler reads it once per
// stream and runs that format's body)
struct MixedRows {
    static constexpr bool kGathered = true, kMixed = true;
    const int32_t *ids; int first; const uint8_t *fmt;
    MWW_HD int io(int s) const { return ids[s] - first; }
    MWW_HD int hist(int s) const { return ids[s]; }
    MWW_HD int format(int s) const { return fmt[ids[s]]; }
};

// Mixed rows of a call of n16 at counter t16 (per-stream rates): the bytes the widest row of streams [first, first + n)
// holds, D_s * format_bytes(f_s), rates[s] one of kResampleRates.  The staged paths copy each tile's rows this wide.
inline long long mixed_rows_width(const int32_t *rates, const uint8_t *formats, int first, int n, long long t16, int n16) {
    constexpr int kRates = (int)(sizeof kResampleRates / sizeof kResampleRates[0]);
    long long D[kRates];
    for (int i = 0; i < kRates; ++i) {
        const int g = resample_gcd(16000, kResampleRates[i]), L = 16000 / g, M = kResampleRates[i] / g;
        D[i] = resample_inputs(t16 + n16, L, M) - resample_inputs(t16, L, M);
    }
    long long w = 0;
    for (int s = first; s < first + n; ++s) {
        int i = 0;
        while (i + 1 < kRates && kResampleRates[i] != rates[s]) ++i;
        const long long b = D[i] * format_bytes(formats[s]);
        w = b > w ? b : w;
    }
    return w;
}

// Output q of a call: t = t0 + q M upsampled samples past the call's first input, newest input k = floor(t / L), phase
// p = t mod L, and y = sat16((sum_i table[p][i] x(k - i) + 2^14) >> 15) over i < T.  x(j) is the call's input j for j >= 0 and
// history[H + j] before it.  X is any accessor with int32_t operator()(int j).
template <typename X>
MWW_HD int16_t resample_output(const int16_t *table, int pitch, int T, int L, int M, int t0, int q, const X &x) {
    const int t = t0 + q * M;
    const int k = t / L;
    const int16_t *h = table + (t - k * L) * pitch;
    int32_t a0 = 0, a1 = 0;
    int i = 0;
    for (; i + 1 < T; i += 2) {
        a0 += (int32_t)h[i] * x(k - i);
        a1 += (int32_t)h[i + 1] * x(k - i - 1);
    }
    if (i < T) a0 += (int32_t)h[i] * x(k - i);
    const long long s = ((long long)a0 + a1 + 16384) >> 15;
    return (int16_t)(s > 32767 ? 32767 : (s < -32768 ? -32768 : s));
}

}  // namespace mww
