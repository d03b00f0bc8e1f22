// mww_detector_groups.h -- grouped detection (include/mww.h, "grouped detection"): the bodies of the rule that merges the
// detections of a group's rows into windows and keeps the best one of each -- the key a candidate is offered with, the offer,
// and the close that applies the rule's steps 1 to 3 to one group at the end of an update.  The kernels are in
// mww_detector_groups.cu; the per-row bodies they run are the detectors' own (mww_detector.h, mww_detector_models.h).
//
// CUDA-free apart from MWW_HD and the offer's device branch, so that tests/emul_detector_groups.cc runs the same functions
// on the CPU.
//
// Offer.  The candidates of one update go to the group's pending slot through three atomics: a 128-bit compare-and-swap
// loop that keeps the largest key (sm_90's 16-byte atomicCAS), an atomicMin of the candidate's step index in the call and
// an atomicAdd of the count.  The key orders candidates by the rule's tie levels, so the maximum is the same whatever order
// the offers arrive in:
//   hi = ordered(score) << 32 | ~t           highest score, then the earliest step of the call (t: the step's index in it)
//   lo = ~biased(stream) << 32 | ~row        then the lowest stream id (then the lowest row, for a stream map that repeats)
// Within one update and one group slot the position of a step grows with t (a slot is one model), so "earliest step" is
// "earliest position", and the smallest t fixes p_min.  The key holds no position and no step count: the close rebuilds
// them from t with the call's clock and from the row's `seen` after the call (each row advances by the call's n steps).
#pragma once

#include <stdint.h>

#include "../../include/mww.h"
#include "mww_common.h"
#include "mww_detector_models.h"

namespace mww {

struct alignas(16) GroupKey {
    unsigned long long hi = 0, lo = 0;       // 0, 0: no candidate (every candidate's hi is above 2^32)
};

// what one update offered to a group: the best key, the smallest t and the number of candidates; zeroed (tmin all ones)
// again by the close
struct alignas(16) GroupPending {
    GroupKey best;
    uint32_t count = 0, tmin = 0xffffffffu;
    uint32_t pad[2] = {0, 0};
};

// what the grouped kernels get beside the detector's own arguments: the groups, each group slot's pending offers and window,
// and what a grouped detector stores beside each event (its position, group and candidates).  A slot is a group (plain) or a
// (group, WAKE model) pair, g n_wake + w (models; wake_of[k] = w for WAKE model k).
struct GroupArgs {
    const int32_t *groups = nullptr;         // [rows (plain) or global streams (models)], -1: none
    GroupPending *pending = nullptr;         // [n_slots]
    mww_group_window *windows = nullptr;     // [n_slots]
    long long *positions = nullptr;          // [capacity], as a timed detector's
    int32_t *ev_group = nullptr, *ev_candidates = nullptr;   // [capacity]
    long long window = 0;                    // W
    int n_slots = 0, n_wake = 1;
    int8_t wake_of[kDetectMaxModels] = {};
};

MWW_HD bool group_key_less(const GroupKey &a, const GroupKey &b) { return a.hi < b.hi || (a.hi == b.hi && a.lo < b.lo); }

// float bits in an order where a larger unsigned value is a larger float
MWW_HD uint32_t group_ordered(float f) {
#if defined(__CUDA_ARCH__)
    const uint32_t u = __float_as_uint(f);
#else
    uint32_t u;
    __builtin_memcpy(&u, &f, 4);
#endif
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
MWW_HD float group_unordered(uint32_t u) {
    u = (u & 0x80000000u) ? (u & 0x7fffffffu) : ~u;
#if defined(__CUDA_ARCH__)
    return __uint_as_float(u);
#else
    float f;
    __builtin_memcpy(&f, &u, 4);
    return f;
#endif
}

MWW_HD GroupKey group_key(float score, int t, int32_t stream, int row) {
    GroupKey k;
    k.hi = (unsigned long long)group_ordered(score) << 32 | (uint32_t)~(uint32_t)t;
    k.lo = (unsigned long long)(uint32_t)~((uint32_t)stream ^ 0x80000000u) << 32 | (uint32_t)~(uint32_t)row;
    return k;
}
MWW_HD float group_key_score(const GroupKey &k) { return group_unordered((uint32_t)(k.hi >> 32)); }
MWW_HD int group_key_t(const GroupKey &k) { return (int)~(uint32_t)k.hi; }
MWW_HD int32_t group_key_stream(const GroupKey &k) { return (int32_t)(~(uint32_t)(k.lo >> 32) ^ 0x80000000u); }
MWW_HD int group_key_row(const GroupKey &k) { return (int)~(uint32_t)k.lo; }

// one candidate into a group's pending slot.  The swap is sm_90's atom.cas.b128 in inline PTX: the 16-byte atomicCAS
// template takes its operands by address, which put them in local memory
MWW_HD void group_offer(GroupPending *p, const GroupKey &k, int t) {
#if defined(__CUDA_ARCH__)
    atomicAdd(&p->count, 1u);
    atomicMin(&p->tmin, (uint32_t)t);
    // the swap loop in PTX, so that its 128-bit registers stay inside it (written in C++ around the 16-byte atomicCAS, the
    // loop made ptxas spill the kernels' other registers)
    asm volatile("{\n\t"
                 ".reg .b128 c, v, o;\n\t.reg .b64 ch, cl, oh, ol;\n\t.reg .pred p, q, r;\n\t"
                 "mov.b64 ch, 0;\n\tmov.b64 cl, 0;\n\t"
                 "mov.b128 v, {%0, %1};\n"
                 "GROUP_OFFER_LOOP:\n\t"
                 "setp.lt.u64 p, ch, %0;\n\tsetp.eq.u64 q, ch, %0;\n\tsetp.lt.and.u64 r, cl, %1, q;\n\tor.pred p, p, r;\n\t"
                 "@!p bra GROUP_OFFER_DONE;\n\t"
                 "mov.b128 c, {ch, cl};\n\t"
                 "atom.global.cas.b128 o, [%2], c, v;\n\t"
                 "mov.b128 {oh, ol}, o;\n\t"
                 "setp.eq.u64 q, oh, ch;\n\tsetp.eq.and.u64 q, ol, cl, q;\n\t"
                 "mov.b64 ch, oh;\n\tmov.b64 cl, ol;\n\t"
                 "@!q bra GROUP_OFFER_LOOP;\n"
                 "GROUP_OFFER_DONE:\n\t}"
                 :: "l"(k.hi), "l"(k.lo), "l"(&p->best) : "memory");
#else
    p->count += 1;
    if ((uint32_t)t < p->tmin) p->tmin = (uint32_t)t;
    if (group_key_less(p->best, k)) p->best = k;
#endif
}

// an event the close stores: the winner's own stream, step, score and position, its group and the candidates merged into it
struct GroupEvent {
    long long sample = 0, step = 0;
    int32_t stream = 0, candidates = 0;
    float score = 0.f;
    float level = 0.f;                       // an arbitrated detector's (mww_group_arbitration.h); not read otherwise
};

MWW_HD GroupEvent group_window_event(const mww_group_window &w) {
    GroupEvent e;
    e.sample = w.sample; e.step = w.step; e.stream = w.stream; e.candidates = w.candidates; e.score = w.score;
    return e;
}

// what one close emits, in this order: the window step 1 closed (before this update's candidates) and the one step 3 closed
struct GroupClosed {
    bool first = false, second = false;
    GroupEvent e1, e2;
};

// whether an update's best replaces the window's: always into a closed window; into an open one when it is better, a tie keeping
// the earlier candidate -- a higher score, or (kLevel, group arbitration) a higher level, then a higher score
template <bool kLevel>
MWW_HD bool group_takes(const mww_group_window &w, const GroupEvent &best, float w_level) {
    if constexpr (kLevel) {
        const uint32_t b = group_ordered(best.level), o = group_ordered(w_level);
        return !w.open || b > o || (b == o && group_ordered(best.score) > group_ordered(w.score));
    } else {
        return !w.open || group_ordered(best.score) > group_ordered(w.score);
    }
}

// The rule's steps 1 to 3 for one group at the end of an update.  n: the candidates of this update (best: the best of them,
// with its position and step; p_min: their smallest position).  has_first: the update had a step (a models update in which
// this model ran no step has none, and step 1 is skipped: step 3 decides alone).  a, E: the update's a_u and E_u; W: the
// window.  A flush is E = the largest value, has_first false, n 0.  kLevel (group arbitration): *w_level is the open window's
// level, compared first and carried into the emitted events.
template <bool kLevel = false>
MWW_HD GroupClosed group_close(mww_group_window &w, uint32_t n, const GroupEvent &best, long long p_min, bool has_first, long long a,
                               long long E, long long W, float *w_level = nullptr) {
    GroupClosed c;
    if (w.open && has_first && a >= w.deadline) {
        c.first = true; c.e1 = group_window_event(w); w.open = 0;
        if constexpr (kLevel) c.e1.level = *w_level;
    }
    if (n) {
        const bool take = group_takes<kLevel>(w, best, kLevel ? *w_level : 0.f);
        if (!w.open) { w.open = 1; w.deadline = p_min + W; w.candidates = 0; }
        if (take) { w.sample = best.sample; w.step = best.step; w.stream = best.stream; w.score = best.score; }
        if constexpr (kLevel) { if (take) *w_level = best.level; }
        w.candidates += (int32_t)n;
    }
    if (w.open && E >= w.deadline) {
        c.second = true; c.e2 = group_window_event(w); w.open = 0;
        if constexpr (kLevel) c.e2.level = *w_level;
    }
    return c;
}

}  // namespace mww
