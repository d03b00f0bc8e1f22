// emul_detector_groups.cc -- the bodies of grouped detection (microwakeword_b200/csrc/mww_detector_groups.h) on the CPU, for
// tests/test_detector_groups.py: an update's candidates offered to their group slots (group_key, group_offer) in the order
// given, then every slot closed (group_close) with the plain detector's clock, as detector_groups_close_kernel does, and the
// winners appended through a counter that counts past capacity.
#include "../microwakeword_b200/csrc/mww_event_positions.h"
#include "../microwakeword_b200/csrc/mww_detector_groups.h"

using namespace mww;

namespace {

struct Buffer {
    long long *count; int capacity;
    long long *sample, *step; int32_t *stream, *group, *candidates; float *score;
    void put(const GroupEvent &e, int grp) {
        const long long slot = (*count)++;
        if (slot >= capacity) return;
        sample[slot] = e.sample; step[slot] = e.step; stream[slot] = e.stream; score[slot] = e.score; group[slot] = grp;
        candidates[slot] = e.candidates;
    }
};

}  // namespace

extern "C" {

int emul_sizes(int *pending, int *window) {
    *pending = (int)sizeof(GroupPending);
    *window = (int)sizeof(mww_group_window);
    return 0;
}

void emul_pending_init(GroupPending *p, int n) {
    for (int i = 0; i < n; ++i) p[i] = GroupPending{};
}

// One plain update of n steps on the clock (last_end, step_samples): candidate i (slot[i], t[i], score[i], stream[i], row[i])
// is offered, then every slot closes; seen_after[row] is the row's seen after the call.  flush: the close alone, as
// mww_flush_detector_groups.  Returns the events appended.
long long emul_group_update(int n_slots, long long W, GroupPending *pending, mww_group_window *windows, int n_cand, const int32_t *slot,
                            const int32_t *t, const float *score, const int32_t *stream, const int32_t *row, const long long *seen_after,
                            long long last_end, long long step_samples, int n, int flush, long long *count, int capacity, long long *o_sample,
                            long long *o_step, int32_t *o_stream, float *o_score, int32_t *o_group, int32_t *o_candidates) {
    for (int i = 0; i < n_cand; ++i) group_offer(&pending[slot[i]], group_key(score[i], t[i], stream[i], row[i]), t[i]);
    Buffer buf{count, capacity, o_sample, o_step, o_stream, o_group, o_candidates, o_score};
    const long long before = *count;
    for (int s = 0; s < n_slots; ++s) {
        const GroupPending p = pending[s];
        GroupEvent best;
        long long p_min = 0;
        if (p.count) {
            const int tb = group_key_t(p.best);
            best.stream = group_key_stream(p.best);
            best.score = group_key_score(p.best);
            best.sample = event_step_end(last_end, step_samples, n, tb);
            best.step = seen_after[group_key_row(p.best)] - n + tb;
            p_min = event_step_end(last_end, step_samples, n, (int)p.tmin);
            pending[s] = GroupPending{};
        }
        const GroupClosed c = group_close(windows[s], p.count, best, p_min, !flush && n > 0, n > 0 ? event_step_end(last_end, step_samples, n, 0) : 0,
                                          flush ? 0x7fffffffffffffffLL : last_end + step_samples, W);
        if (c.first) buf.put(c.e1, s);
        if (c.second) buf.put(c.e2, s);
    }
    return *count - before;
}

}  // extern "C"
