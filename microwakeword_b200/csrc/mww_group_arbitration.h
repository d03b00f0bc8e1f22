// mww_group_arbitration.h -- household arbitration (include/mww.h, "group arbitration"): the bodies of the rule that picks a
// group's winner by the level of the wake word over its noise floor -- the spans a candidate is measured over, the energy and
// level arithmetic, the key a candidate is offered with, and the close of one group slot.  The kernels are in
// mww_group_arbitration.cu; the offer and the window steps are grouped detection's (mww_detector_groups.h).
//
// CUDA-free apart from MWW_HD and the device branches of the arithmetic, so that tests/emul_group_arbitration.cc runs the same
// functions on the CPU (built with -ffp-contract=off: every double operation is rounded on its own, as __dmul_rn and friends
// are on the device).
//
// Key.  hi = ordered(level) << 32 | ordered(score), lo = ~t << 32 | ~id: the highest level, then the highest score, then the
// earliest step of the call, then the lowest id -- the row (plain detector) or the global stream (models detector).  It fits
// the offer's 128-bit compare-and-swap, so the maximum is the same whatever order the offers arrive in.
#pragma once

#include <stdint.h>

#include "mww_detector_groups.h"

namespace mww {

constexpr int kArbitrationMinSamples = 480, kArbitrationMaxSamples = 1 << 20;

// what the arbitrated kernels get beside the grouped ones' arguments: the source handle's history as of the update (ring
// [n_streams][capacity], `seen` its samples_seen), the two span lengths, each group slot's best level, and each event slot's
// level (NaN for an event of a row of group -1)
struct ArbitrationArgs {
    const int16_t *ring = nullptr;
    long long seen = 0;
    int capacity = 0;
    int speech = 0, noise = 0;                // Ls, Ln
    float *levels = nullptr;                  // [n_slots]
    float *ev_level = nullptr;                // [detector capacity]
};

MWW_HD GroupKey arbitration_key(float level, float score, int t, int id) {
    GroupKey k;
    k.hi = (unsigned long long)group_ordered(level) << 32 | group_ordered(score);
    k.lo = (unsigned long long)(uint32_t)~(uint32_t)t << 32 | (uint32_t)~(uint32_t)id;
    return k;
}
MWW_HD float arbitration_key_level(const GroupKey &k) { return group_unordered((uint32_t)(k.hi >> 32)); }
MWW_HD float arbitration_key_score(const GroupKey &k) { return group_unordered((uint32_t)k.hi); }
MWW_HD int arbitration_key_t(const GroupKey &k) { return (int)~(uint32_t)(k.lo >> 32); }
MWW_HD int arbitration_key_id(const GroupKey &k) { return (int)~(uint32_t)k.lo; }

// The positions of a candidate at P that the ring holds: [lo, hi) = [P - Ls - Ln, P) cut to [S - C, S).  Positions outside it
// read as zeros; hi <= lo when none is held.  The noise span is the part below P - Ls, the speech span the rest.
struct ArbitrationSpan {
    long long lo, hi, split;                  // split = P - Ls
};
MWW_HD ArbitrationSpan arbitration_span(long long P, int Ls, int Ln, long long S, int C) {
    ArbitrationSpan s;
    s.split = P - Ls;
    s.lo = P - Ls - Ln > S - C ? P - Ls - Ln : S - C;
    s.hi = P < S ? P : S;
    return s;
}

// the mean-removed power of a span of L samples with q = sum x^2 (exact below 2^53) and r = sum x: (q - r r / L) / L
MWW_HD double arbitration_energy(unsigned long long q, long long r, int L) {
    const double dq = (double)q, dr = (double)r, dl = (double)L;
#if defined(__CUDA_ARCH__)
    return __ddiv_rn(__dsub_rn(dq, __ddiv_rn(__dmul_rn(dr, dr), dl)), dl);
#else
    return (dq - dr * dr / dl) / dl;
#endif
}

// the level: (e_speech + 1) / (e_noise + 1), rounded to the nearest float; one LSB^2 of floor, so all-zero noise divides by 1
MWW_HD float arbitration_level(double e_speech, double e_noise) {
#if defined(__CUDA_ARCH__)
    return __double2float_rn(__ddiv_rn(__dadd_rn(e_speech, 1.0), __dadd_rn(e_noise, 1.0)));
#else
    return (float)((e_speech + 1.0) / (e_noise + 1.0));
#endif
}

// One arbitrated slot's close: its pending offers resolved with the call's clock (pos(t): the position of step t; seen(id):
// the row's seen after the call, of the row or stream id; stream(id): the event's stream), grouped detection's steps 1 to 3
// with the level order, and the pending slot cleared.  n: the call's steps (0 for a flush); E: E_u.
template <typename Pos, typename Seen, typename Stream>
MWW_HD GroupClosed arbitration_close_slot(GroupPending *pending, mww_group_window *windows, float *levels, long long W, int s, int n,
                                          const Pos &pos, const Seen &seen, const Stream &stream, long long E, bool flush) {
    const GroupPending p = pending[s];
    GroupEvent best;
    long long p_min = 0;
    if (p.count) {
        const int t = arbitration_key_t(p.best), id = arbitration_key_id(p.best);
        best.stream = stream(id);
        best.score = arbitration_key_score(p.best);
        best.level = arbitration_key_level(p.best);
        best.sample = pos(t);
        best.step = seen(id) - n + t;
        p_min = pos((int)p.tmin);
        pending[s] = GroupPending{};
    }
    mww_group_window w = windows[s];
    float level = levels[s];
    const GroupClosed c = group_close<true>(w, p.count, best, p_min, !flush && n > 0, n > 0 ? pos(0) : 0, flush ? 0x7fffffffffffffffLL : E, W,
                                            &level);
    if (p.count || c.first || c.second) { windows[s] = w; levels[s] = level; }
    return c;
}

}  // namespace mww
