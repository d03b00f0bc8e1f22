// mww_detector.h -- the streaming detector (mww_detector_*, include/mww.h): the per-row rule in the two forms
// detector_update_kernel runs it (mww_detector.cu).  CUDA-free apart from MWW_HD, so that tests/emul_detector.cc runs
// the same functions on the CPU.
//
// Definition.  A row consumes probabilities p[0], p[1], ...; with avg[i] = mean(p[i .. i + window)) in float32, for
// i = 0, 1, ...: cooldown = max(cooldown - 1, 0); if cooldown == 0 and (double)avg[i] > cutoff the row fires (step
// i + window - 1, score avg[i]) and cooldown = cooldown_slices.  That is false_accept_kernel (mww_detect.cu) on the
// concatenation of everything the row was given; the state carried between calls is the last window - 1 probabilities,
// the count of probabilities seen and the cooldown.  In per-row mode (mww_set_detector_cutoffs) `cutoff` is the row's
// c_r, which the _at and _from forms of the rule take as an argument; nothing else changes.
#pragma once

#include <stdint.h>

#include "../../include/mww.h"
#include "mww_common.h"

namespace mww {

constexpr int kDetectorMaxWindow = 32;      // one 32-step pass of the warp form holds every window's history
// calls of at least this many steps per row take the warp form.  Measured (tools/detector_time.py, H100 SXM at 700 W,
// window 5): the thread form's time grows with every step, the warp form's with every pass of 32, and they cross near
// 48 steps, at 65 536 rows (state in L2) and at 4 M rows (state in HBM) alike (DESIGN.md section 4).
constexpr int kDetectorWarpMinSteps = 48;

struct DetectorRule {
    int window = 5, cooldown_slices = 25;
    double cutoff = 0.5;
};

// what the update and reset kernels get: per-row state as struct-of-arrays (hist [window - 1][n_rows], so a thread per
// row reads and writes it coalesced), the event buffer, its counter and the fired-id list
struct DetectorArgs {
    DetectorRule rule;
    int n_rows = 0, capacity = 0;
    float *hist = nullptr;
    long long *seen = nullptr;
    int32_t *cooldown = nullptr;
    const int32_t *stream_ids = nullptr;      // row -> event.stream, nullptr: the row index
    unsigned long long *count = nullptr;
    mww_event *events = nullptr;
    int32_t *fired = nullptr;
};

// float32 add and divide, rounded to nearest and never contracted: NumPy's float32 mean is a sequential sum and one division
MWW_HD float det_add(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fadd_rn(a, b);
#else
    return a + b;
#endif
}
MWW_HD float det_div(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fdiv_rn(a, b);
#else
    return a / b;
#endif
}
MWW_HD int det_lowest_bit(unsigned m) {
#if defined(__CUDA_ARCH__)
    return __ffs((int)m) - 1;
#else
    return __builtin_ctz(m);
#endif
}

// window_mean of mww_detect.cu over x(newest - window + 1) .. x(newest), oldest first.  X: float operator()(int) const.
template <typename X>
MWW_HD float detector_window_mean(const X &x, int newest, int window) {
    float s = x(newest - window + 1);
    for (int j = newest - window + 2; j <= newest; ++j) s = det_add(s, x(j));
    return det_div(s, (float)window);
}

// a cutoff held as a value
struct CutoffValue {
    double c = 0.0;
    MWW_HD double get() const { return c; }
};

// the rule at one moving-average index against a cutoff (C: double get() const; the rule's, or the row's in per-row mode),
// which is read only once the cooldown has run out: true when it fires
template <typename C>
MWW_HD bool detector_tick_from(const DetectorRule &r, const C &cutoff, float avg, int &cooldown) {
    cooldown = cooldown > 0 ? cooldown - 1 : 0;
    if (cooldown != 0 || !((double)avg > cutoff.get())) return false;
    cooldown = r.cooldown_slices;
    return true;
}
MWW_HD bool detector_tick_at(const DetectorRule &r, double cutoff, float avg, int &cooldown) {
    return detector_tick_from(r, CutoffValue{cutoff}, avg, cooldown);
}
MWW_HD bool detector_tick(const DetectorRule &r, float avg, int &cooldown) { return detector_tick_at(r, r.cutoff, avg, cooldown); }

// Thread form: one row takes one probability.  `seen` counts the probabilities before this one (the caller adds one
// afterwards).  The history is streamed, never held: entry j is read, summed and written back to j - 1, so a window of
// any length needs no array.  H: float get(int) const, void set(int, float) over the row's window - 1 entries.
template <typename H>
MWW_HD bool detector_step_at(H &hist, const DetectorRule &r, double cutoff, long long seen, int &cooldown, float p, float *score) {
    const int w = r.window;
    float s = p;
    if (w > 1) {
        s = hist.get(0);
        for (int j = 1; j < w - 1; ++j) {
            const float v = hist.get(j);
            s = det_add(s, v);
            hist.set(j - 1, v);
        }
        s = det_add(s, p);
        hist.set(w - 2, p);
    }
    if (seen + 1 < w) return false;              // warming up: the sum holds entries from before the reset
    const float avg = det_div(s, (float)w);
    if (!detector_tick_at(r, cutoff, avg, cooldown)) return false;
    *score = avg;
    return true;
}
template <typename H>
MWW_HD bool detector_step(H &hist, const DetectorRule &r, long long seen, int &cooldown, float p, float *score) {
    return detector_step_at(hist, r, r.cutoff, seen, cooldown, p, score);
}

// Warp form: a pass covers n <= 32 consecutive steps of one row, lane i forming the average whose newest probability is
// step i of the pass.  Whether an average exceeds the cutoff does not depend on the cooldown, so the lanes find the
// candidates together (a ballot) and only the chain is walked in order, over the candidate mask, by every lane alike.
// The cooldown ticks on every step that has a full window -- steps `first` .. n - 1 of the pass -- so between candidates it
// advances by the gap.  candidates: bit i set when step i has a full window and avg > cutoff.  Returns the steps that fire.
MWW_HD unsigned detector_chain_pass(const DetectorRule &r, unsigned candidates, int first, int n, int &cooldown) {
    unsigned fired = 0;
    int pos = first;                             // the next step whose tick has not been applied
    for (unsigned m = candidates; m; m &= m - 1) {
        const int j = det_lowest_bit(m);
        const int left = cooldown - (j - pos + 1);
        pos = j + 1;
        if (left > 0) { cooldown = left; continue; }
        fired |= 1u << j;
        cooldown = r.cooldown_slices;
    }
    if (pos < n) cooldown = cooldown - (n - pos) > 0 ? cooldown - (n - pos) : 0;
    return fired;
}

// first step of a pass that has a full window, for a pass whose step 0 is the row's probability number `seen`; n when none has
MWW_HD int detector_first_full(long long seen, int window, int n) {
    const long long f = (long long)(window - 1) - seen;
    return f <= 0 ? 0 : (f < n ? (int)f : n);
}

}  // namespace mww
