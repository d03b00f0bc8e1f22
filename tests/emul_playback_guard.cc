// emul_playback_guard.cc -- the bodies of the playback guard (microwakeword_b200/csrc/mww_playback.h) on the CPU, for
// tests/test_playback_guard.py: a write call as the host plans it and the write kernel runs it (the mirror, the device map and
// heads, the ring), the read of the slots kernel, a check's slots and heard flags, and the decision.
#include <vector>

#include "../microwakeword_b200/csrc/mww_playback.h"

using namespace mww;

extern "C" {

int emul_sizes(int *rule, int *desc) {
    *rule = (int)sizeof(mww_playback_rule);
    *desc = (int)sizeof(mww_playback_guard_desc);
    return 0;
}

// One write call: playback_plan from the mirror (row_of, stream_of, head), every job as playback_write_kernel runs it on ring
// [rows][C] and the device map dev_row_of / dev_head, then playback_commit.  Returns the number of jobs, or -1 (nothing changed).
int emul_write(const int32_t *ids, const long long *starts, int n, const int16_t *audio, int n_samples, long long seen, int C, int rows,
               int n_streams, int32_t *row_of, int32_t *stream_of, long long *head, int16_t *ring, int32_t *dev_row_of, long long *dev_head) {
    std::vector<char> listed(n_streams, 0);
    for (int i = 0; i < n; ++i) listed[ids[i]] = 1;
    std::vector<PlaybackJob> jobs(n_streams + rows);
    const int n_jobs = playback_plan(ids, starts, n, seen, C, rows, row_of, stream_of, head, listed.data(), jobs.data());
    if (n_jobs < 0) return -1;
    for (int j = 0; j < n_jobs; ++j) {
        const PlaybackJob &job = jobs[j];
        if (job.row < 0) { dev_row_of[job.stream] = -1; continue; }
        const PlaybackWrite p = playback_write_plan(job.start, n_samples, job.head, C);
        for (long long k = 0; k < p.len; ++k) {
            const long long q = p.span0 + k;
            ring[(long long)job.row * C + playback_mod(q, C)] = playback_write_value(audio + (long long)j * n_samples, job.start, q);
        }
        dev_row_of[job.stream] = job.row;
        dev_head[job.row] = p.head;
    }
    playback_commit(jobs.data(), n, n_samples, seen, C, rows, row_of, stream_of, head);
    return n_jobs;
}

// the read of the slots kernel: out [n][L] row i = pb of ids[i] over [ends[i] - min_delay - L, ends[i] - min_delay)
void emul_read(const int32_t *ids, const long long *ends, int n, int L, long long min_delay, int n_streams, int C, const int16_t *ring,
               const int32_t *dev_row_of, const long long *dev_head, int16_t *out) {
    for (int i = 0; i < n; ++i) {
        const bool listed = ids[i] >= 0 && ids[i] < n_streams;
        const int32_t r = listed ? dev_row_of[ids[i]] : -1;
        const long long w = r >= 0 ? dev_head[r] : 0, r0 = playback_ref_end(ends[i], min_delay) - L;
        for (int k = 0; k < L; ++k) out[(long long)i * L + k] = playback_read_one(ring + (long long)(r >= 0 ? r : 0) * C, C, r >= 0, w, r0 + k);
    }
}

// heard flags of n slots given as ids and ends (a check of streams)
void emul_heard(const int32_t *ids, const long long *ends, int n, int L, long long min_delay, int n_streams, int C, long long seen,
                const int32_t *dev_row_of, const long long *dev_head, int32_t *heard) {
    for (int i = 0; i < n; ++i) {
        const PlaybackSlot s = playback_slot_streams(ids[i], ends[i]);
        const bool listed = s.sid >= 0 && s.sid < n_streams;
        const int32_t r = listed ? dev_row_of[s.sid] : -1;
        const long long r0 = playback_ref_end(s.end, min_delay) - L;
        heard[i] = playback_heard(s.sid, n_streams, r >= 0, r >= 0 ? dev_head[r] : 0, r0, seen, C) ? 1 : 0;
    }
}

// playback_slot_detector of every slot: sid and end
void emul_slots_detector(int capacity, long long count, const mww_event *events, const long long *positions, int model, long long post, long long seen,
                         int32_t *sid, long long *end) {
    for (int i = 0; i < capacity; ++i) {
        const PlaybackSlot s = playback_slot_detector(i, count, capacity, events, positions, model, post, seen);
        sid[i] = s.sid;
        end[i] = s.end;
    }
}

void emul_decide(int n, const int32_t *heard, const float *scores, double cutoff, const int32_t *confirmed, float *out_scores, int32_t *flagged,
                 int32_t *passed) {
    for (int i = 0; i < n; ++i) {
        const PlaybackOut o = playback_decide(heard[i] != 0, scores[i], cutoff, confirmed[i]);
        out_scores[i] = o.score; flagged[i] = o.flagged; passed[i] = o.passed;
    }
}

}  // extern "C"
