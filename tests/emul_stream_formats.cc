// tests/emul_stream_formats.cc -- TEST INFRASTRUCTURE: the resampler stage of a handle with per-stream rates and per-stream
// sample formats (mww_set_stream_formats, the _mixed entry points) on the CPU, for tests/test_stream_formats.py.  It plans a
// call as mww_capi.cu's run_rates_tile does (one sorted member list per rate, tile_members per tile, t0 from N(t)), maps rows
// with MixedRows of microwakeword_b200/csrc/mww_resample.h and dispatches on each member's format once, as resample_kernel
// does, to a body that reads the row's samples with the product's pcm16 (mww_frontend_dev.cuh): the identity plan for 16 kHz
// members, resample_output and the history update for every other rate.  mixed_rows_width is the staged paths' tile width.
#include <vector>

#include "../microwakeword_b200/csrc/mww_frontend_dev.cuh"
#include "../microwakeword_b200/csrc/mww_resample.h"
#include "../microwakeword_b200/csrc/mww_streams.h"

using namespace mww;

namespace {
template <typename T>
struct CallInput {
    const int16_t *hist; const T *x; int H;
    int32_t operator()(int j) const { return j >= 0 ? (int32_t)pcm16(x[j]) : hist[H + j]; }
};

// one CTA's stream: x its row (samples of type T), hs its history, ys its 16 kHz output
template <typename T>
void stream_body(const ResamplePlan &P, const int16_t *table, int t0, int n_in, int n16, const T *x, int16_t *hs, int16_t *ys) {
    if (P.T == 0) {
        for (int q = 0; q < n16; ++q) ys[q] = pcm16(x[q]);
        return;
    }
    const CallInput<T> in{hs, x, P.H};
    for (int q = 0; q < n16; ++q) ys[q] = resample_output(table, P.pitch, P.T, P.L, P.M, t0, q, in);
    std::vector<int16_t> next((size_t)P.H);
    for (int j = 0; j < P.H; ++j) next[j] = (int16_t)in(n_in - P.H + j);
    for (int j = 0; j < P.H; ++j) hs[j] = next[j];
}
}  // namespace

extern "C" {

// One call of n16 16 kHz samples on S streams at counter t (even), streams cut into tiles of `tile`.  rates [S] and formats
// [S] (kFormat* codes); hist [S][hist_stride] is read and moved on (each stream its first H); x holds S rows of pitch_bytes
// bytes, row s D_s samples of its format; y [S][n16].  Returns 0, or -1 for a rate outside the list.
int emul_formats_call(const int32_t *rates, const uint8_t *formats, int S, int16_t *hist, int hist_stride, const uint8_t *x,
                      long long pitch_bytes, long long t, int n16, int tile, int16_t *y) {
    for (int r : kResampleRates) {
        ResamplePlan P;
        resample_plan(r, &P);
        std::vector<int32_t> taps((size_t)(P.n_taps > 0 ? P.n_taps : 1));
        if (P.n_taps > 0 && !resample_taps(P, taps.data())) return -2;
        std::vector<int16_t> table((size_t)P.L * (P.pitch > 0 ? P.pitch : 1));
        if (P.n_taps > 0) resample_table(P, taps.data(), table.data());
        std::vector<int32_t> ids;
        for (int s = 0; s < S; ++s) {
            bool listed = false;
            for (int q : kResampleRates) listed = listed || q == rates[s];
            if (!listed) return -1;
            if (rates[s] == r) ids.push_back(s);
        }
        const long long seen = resample_inputs(t, P.L, P.M);
        const int n_in = (int)(resample_inputs(t + n16, P.L, P.M) - seen), t0 = resample_t0(seen, P.L, P.M);
        for (int first = 0; first < S; first += tile) {
            const int n = S - first < tile ? S - first : tile;
            int a = 0, b = 0;
            tile_members(ids.data(), (int)ids.size(), first, n, &a, &b);
            if (b == a || n_in <= 0) continue;
            const MixedRows rows{ids.data() + a, first, formats};
            const uint8_t *x_tile = x + (size_t)first * pitch_bytes;
            int16_t *y_tile = y + (size_t)first * n16;
            for (int i = 0; i < b - a; ++i) {
                const uint8_t *xs = x_tile + (size_t)rows.io(i) * pitch_bytes;
                int16_t *hs = hist + (size_t)rows.hist(i) * hist_stride;
                int16_t *ys = y_tile + (size_t)rows.io(i) * n16;
                switch (rows.format(i)) {
                case kFormatUlaw: stream_body(P, table.data(), t0, n_in, n16, reinterpret_cast<const Ulaw8 *>(xs), hs, ys); break;
                case kFormatAlaw: stream_body(P, table.data(), t0, n_in, n16, reinterpret_cast<const Alaw8 *>(xs), hs, ys); break;
                case kFormatF32: stream_body(P, table.data(), t0, n_in, n16, reinterpret_cast<const float *>(xs), hs, ys); break;
                default: stream_body(P, table.data(), t0, n_in, n16, reinterpret_cast<const int16_t *>(xs), hs, ys); break;
                }
            }
        }
    }
    return 0;
}

long long emul_mixed_rows_width(const int32_t *rates, const uint8_t *formats, int first, int n, long long t, int n16) {
    return mixed_rows_width(rates, formats, first, n, t, n16);
}

int emul_format_bytes(int f) { return format_bytes(f); }

}  // extern "C"
