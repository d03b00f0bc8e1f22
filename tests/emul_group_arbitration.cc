// emul_group_arbitration.cc -- the bodies of group arbitration (microwakeword_b200/csrc/mww_group_arbitration.h) on the CPU, for
// tests/test_group_arbitration.py, built with -ffp-contract=off as the header asks: a candidate's level from a history ring
// (arbitration_span, arbitration_energy, arbitration_level, one sample at a time where the kernel moves 8), and an update's
// candidates offered to their group slots (arbitration_key, group_offer) in the order given, then every slot closed
// (arbitration_close_slot) with the plain detector's clock, as detector_arbitrated_close_kernel does, and the winners appended
// through a counter that counts past capacity.
#include "../microwakeword_b200/csrc/mww_event_positions.h"
#include "../microwakeword_b200/csrc/mww_history.h"
#include "../microwakeword_b200/csrc/mww_group_arbitration.h"

using namespace mww;

extern "C" {

int emul_sizes(int *pending, int *window, int *key) {
    *pending = (int)sizeof(GroupPending);
    *window = (int)sizeof(mww_group_window);
    *key = (int)sizeof(GroupKey);
    return 0;
}

void emul_pending_init(GroupPending *p, int n) {
    for (int i = 0; i < n; ++i) p[i] = GroupPending{};
}

// levels[i] of a candidate of stream ids[i] at P[i] over the ring [n_streams][C] after S samples
void emul_levels(const int16_t *ring, int C, long long S, const int32_t *ids, const long long *P, int n, int Ls, int Ln, float *levels) {
    for (int i = 0; i < n; ++i) {
        const ArbitrationSpan sp = arbitration_span(P[i], Ls, Ln, S, C);
        unsigned long long qs = 0, qn = 0;
        long long rs = 0, rn = 0;
        for (long long p = sp.lo; p < sp.hi; ++p) {
            const int x = ring[(long long)ids[i] * C + history_mod(p, C)];
            if (p >= sp.split) { qs += (unsigned long long)(x * x); rs += x; }
            else { qn += (unsigned long long)(x * x); rn += x; }
        }
        levels[i] = arbitration_level(arbitration_energy(qs, rs, Ls), arbitration_energy(qn, rn, Ln));
    }
}

// the energy of one span from its sums, for the arithmetic's edges
double emul_energy(unsigned long long q, long long r, int L) { return arbitration_energy(q, r, L); }

// One plain update of n steps on the clock (last_end, step_samples): candidate i (slot[i], t[i], level[i], score[i], row[i]) is
// offered, then every slot closes; seen_after[row] is the row's seen after the call and stream_of[row] its stream.  flush: the
// close alone, as mww_flush_detector_groups.  Returns the events appended.
long long emul_arbitrated_update(int n_slots, long long W, GroupPending *pending, mww_group_window *windows, float *w_levels, int n_cand,
                                 const int32_t *slot, const int32_t *t, const float *level, const float *score, const int32_t *row,
                                 const int32_t *stream_of, const long long *seen_after, long long last_end, long long step_samples, int n,
                                 int flush, long long *count, int capacity, long long *o_sample, long long *o_step, int32_t *o_stream,
                                 float *o_score, int32_t *o_group, int32_t *o_candidates, float *o_level) {
    for (int i = 0; i < n_cand; ++i) group_offer(&pending[slot[i]], arbitration_key(level[i], score[i], t[i], row[i]), t[i]);
    const long long before = *count;
    auto put = [&](const GroupEvent &e, int grp) {
        const long long k = (*count)++;
        if (k >= capacity) return;
        o_sample[k] = e.sample; o_step[k] = e.step; o_stream[k] = e.stream; o_score[k] = e.score; o_group[k] = grp;
        o_candidates[k] = e.candidates; o_level[k] = e.level;
    };
    auto pos = [&](int tt) { return event_step_end(last_end, step_samples, n, tt); };
    auto seen = [&](int r) { return seen_after[r]; };
    auto stream = [&](int r) { return stream_of[r]; };
    for (int s = 0; s < n_slots; ++s) {
        const GroupClosed c = arbitration_close_slot(pending, windows, w_levels, W, s, n, pos, seen, stream, last_end + step_samples, flush != 0);
        if (c.first) put(c.e1, s);
        if (c.second) put(c.e2, s);
    }
    return *count - before;
}

}  // extern "C"
