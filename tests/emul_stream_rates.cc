// tests/emul_stream_rates.cc -- TEST INFRASTRUCTURE: the resampler stage of a handle with per-stream rates
// (mww_set_stream_rates) on the CPU, for tests/test_stream_rates.py.  It plans a call as mww_capi.cu's run_rates_tile does
// (one sorted member list per rate, tile_members per tile, t0 from N(t)) and runs resample_kernel's per-stream body with the
// MemberRows row mapping of microwakeword_b200/csrc/mww_resample.h: the identity plan for 16 kHz members, resample_output
// and the history update for every other rate.
#include <vector>

#include "../microwakeword_b200/csrc/mww_resample.h"
#include "../microwakeword_b200/csrc/mww_streams.h"

using namespace mww;

namespace {
struct CallInput {
    const int16_t *hist, *x; int H;
    int32_t operator()(int j) const { return j >= 0 ? x[j] : hist[H + j]; }
};
}  // namespace

extern "C" {

// One call of n16 16 kHz samples on S streams at counter t (even), streams cut into tiles of `tile`.  rates [S]; hist
// [S][hist_stride] is read and moved on (each stream its first H); x [S][pitch] holds stream s's D_s samples; y [S][n16].
// Returns 0, or -1 for a rate outside the list.
int emul_rates_call(const int32_t *rates, int S, int16_t *hist, int hist_stride, const int16_t *x, long long pitch, long long t,
                    int n16, int tile, int16_t *y) {
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
            const MemberRows rows{ids.data() + a, first};
            const int16_t *x_tile = x + (size_t)first * pitch;
            int16_t *y_tile = y + (size_t)first * n16;
            for (int i = 0; i < b - a; ++i) {           // one CTA's stream
                const int16_t *xs = x_tile + (size_t)rows.io(i) * pitch;
                int16_t *hs = hist + (size_t)rows.hist(i) * hist_stride;
                int16_t *ys = y_tile + (size_t)rows.io(i) * n16;
                if (P.T == 0) {
                    for (int q = 0; q < n16; ++q) ys[q] = xs[q];
                    continue;
                }
                const CallInput in{hs, xs, P.H};
                for (int q = 0; q < n16; ++q) ys[q] = resample_output(table.data(), P.pitch, P.T, P.L, P.M, t0, q, in);
                std::vector<int16_t> next((size_t)P.H);
                for (int j = 0; j < P.H; ++j) next[j] = (int16_t)in(n_in - P.H + j);
                for (int j = 0; j < P.H; ++j) hs[j] = next[j];
            }
        }
    }
    return 0;
}

long long emul_rate_inputs(int rate, long long t) {
    ResamplePlan P;
    if (!resample_plan(rate, &P)) return -1;
    return resample_inputs(t, P.L, P.M);
}

int emul_max_history() { return resample_max_history(); }

}  // extern "C"
