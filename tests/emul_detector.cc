// tests/emul_detector.cc -- TEST INFRASTRUCTURE: the streaming detector's rule (microwakeword_b200/csrc/mww_detector.h) run
// on the CPU in both forms of detector_update_kernel, lane by lane for the warp form, for tests/test_detector.py.
#include "../microwakeword_b200/csrc/mww_detector.h"

using namespace mww;

namespace {

struct RowHistory {          // host state is [n_rows][window - 1]: a row's entries are contiguous
    float *h;
    float get(int j) const { return h[j]; }
    void set(int j, float v) { h[j] = v; }
};

struct PassWindow {          // what the kernel's shuffles read: the lanes' registers of this pass and the one before
    const float *cur, *prev;
    float operator()(int i) const { return i >= 0 ? cur[i & 31] : prev[i & 31]; }
};

struct Sink {
    mww_event *events; int max; long long count;
    void add(int row, long long step, float score) {
        if (count < max) events[count] = mww_event{row, 0, step, score, 0};
        ++count;
    }
};

DetectorRule rule(int window, double cutoff, int cooldown_slices) {
    DetectorRule r;
    r.window = window; r.cutoff = cutoff; r.cooldown_slices = cooldown_slices;
    return r;
}

}  // namespace

extern "C" {

int emul_sizeof_event() { return (int)sizeof(mww_event); }
int emul_warp_min_steps() { return kDetectorWarpMinSteps; }

// one update call on host state hist [R][window - 1], seen [R], cooldown [R]; probs [R][pitch].  Events (stream = row) go
// to events[0, max_events) in row-major order of (row, step); returns how many fired.
long long emul_update_thread(int window, double cutoff, int cooldown_slices, float *hist, long long *seen, int32_t *cooldown,
                             const float *probs, int R, int n_steps, long long pitch, mww_event *events, int max_events) {
    const DetectorRule r = rule(window, cutoff, cooldown_slices);
    Sink out{events, max_events, 0};
    for (int row = 0; row < R; ++row) {
        RowHistory h{hist + (long long)row * (window - 1)};
        int cd = cooldown[row];
        for (int t = 0; t < n_steps; ++t) {
            float score = 0.f;
            if (detector_step(h, r, seen[row], cd, probs[row * pitch + t], &score)) out.add(row, seen[row], score);
            ++seen[row];
        }
        cooldown[row] = cd;
    }
    return out.count;
}

// the same call as the warp form runs it: 32-step passes, one average per lane, the chain over the candidate mask
long long emul_update_warp(int window, double cutoff, int cooldown_slices, float *hist, long long *seen, int32_t *cooldown,
                           const float *probs, int R, int n_steps, long long pitch, mww_event *events, int max_events) {
    const DetectorRule r = rule(window, cutoff, cooldown_slices);
    const int w = window;
    Sink out{events, max_events, 0};
    if (n_steps <= 0) return 0;
    for (int row = 0; row < R; ++row) {
        float *h = hist + (long long)row * (w - 1);
        const float *p = probs + row * pitch;
        float cur[32] = {0}, prev[32] = {0};
        for (int lane = 32 - (w - 1); lane < 32; ++lane) prev[lane] = h[lane - (32 - (w - 1))];
        int cd = cooldown[row], n = 0;
        for (int base = 0; base < n_steps; base += 32) {
            n = n_steps - base < 32 ? n_steps - base : 32;
            for (int lane = 0; lane < 32; ++lane) cur[lane] = lane < n ? p[base + lane] : 0.f;
            const PassWindow x{cur, prev};
            const int first = detector_first_full(seen[row] + base, w, n);
            float avg[32];
            unsigned candidates = 0;
            for (int lane = 0; lane < 32; ++lane) {
                avg[lane] = detector_window_mean(x, lane, w);
                if (lane >= first && lane < n && (double)avg[lane] > r.cutoff) candidates |= 1u << lane;
            }
            const unsigned fired = detector_chain_pass(r, candidates, first, n, cd);
            for (int lane = 0; lane < 32; ++lane)
                if ((fired >> lane) & 1u) out.add(row, seen[row] + base + lane, avg[lane]);
            if (base + 32 < n_steps)
                for (int lane = 0; lane < 32; ++lane) prev[lane] = cur[lane];
        }
        const PassWindow x{cur, prev};
        float keep[32];
        for (int lane = 0; lane < w - 1; ++lane) keep[lane] = x(n - (w - 1) + lane);
        for (int lane = 0; lane < w - 1; ++lane) h[lane] = keep[lane];
        seen[row] += n_steps;
        cooldown[row] = cd;
    }
    return out.count;
}

}  // extern "C"
