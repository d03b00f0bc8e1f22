// tests/emul_resample.cc -- TEST INFRASTRUCTURE: the filter design, polyphase table and per-output body of the input-rate
// resampler (microwakeword_b200/csrc/mww_resample.h) run on the CPU with the kernel's index math, for tests/test_resample.py.
#include <vector>

#include "../microwakeword_b200/csrc/mww_resample.h"

using namespace mww;

namespace {
struct CallInput {
    const int16_t *hist, *x; int H;
    int32_t operator()(int j) const { return j >= 0 ? x[j] : hist[H + j]; }
};
}  // namespace

extern "C" {

// out[0..6] = L, M, n_taps, T, H, pitch; 0, or -1 for a rate outside the list
int emul_plan(int rate, int *out) {
    ResamplePlan P;
    if (!resample_plan(rate, &P)) return -1;
    const int v[6] = {P.L, P.M, P.n_taps, P.T, P.H, P.pitch};
    for (int i = 0; i < 6; ++i) out[i] = v[i];
    return 0;
}

// one call of n samples on S streams after `seen` inputs: hist [S][H] is read and moved on, y [S][n_out]; returns n_out
int emul_call(int rate, int16_t *hist, const int16_t *x, int S, int n, long long seen, int16_t *y) {
    ResamplePlan P;
    if (!resample_plan(rate, &P) || P.n_taps == 0) return -1;
    std::vector<int32_t> taps((size_t)P.n_taps);
    if (!resample_taps(P, taps.data())) return -2;
    std::vector<int16_t> table((size_t)P.L * P.pitch);
    resample_table(P, taps.data(), table.data());
    const int n_out = resample_call_outputs(seen, n, P.L, P.M), t0 = resample_t0(seen, P.L, P.M);
    std::vector<int16_t> next((size_t)P.H);
    for (int s = 0; s < S; ++s) {
        int16_t *hs = hist + (size_t)s * P.H;
        const CallInput in{hs, x + (size_t)s * n, P.H};
        for (int q = 0; q < n_out; ++q) y[(size_t)s * n_out + q] = resample_output(table.data(), P.pitch, P.T, P.L, P.M, t0, q, in);
        for (int j = 0; j < P.H; ++j) next[j] = (int16_t)in(n - P.H + j);
        for (int j = 0; j < P.H; ++j) hs[j] = next[j];
    }
    return n_out;
}

}  // extern "C"
