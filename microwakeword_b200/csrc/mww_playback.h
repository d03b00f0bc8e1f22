// mww_playback.h -- the bodies of the playback guard (include/mww.h, "playback guard"): the release of a row, the plan of a
// write into a row, the read of a position, the slots of a check, the heard rule and the decision of a slot.  The kernels are in
// mww_playback.cu; the scoring is the verifier's own pass (mww_verify_capi.cu), run on the guard's verifier.
//
// A row of C samples holds axis positions [w - C, w) for its head w; position p lives in slot p mod C, so a write moves only
// the positions it changes and a read needs no copy of the row.
//
// CUDA-free apart from MWW_HD, so that tests/emul_playback_guard.cc runs the same functions on the CPU.
#pragma once

#include <stdint.h>

#include "../../include/mww.h"
#include "mww_common.h"
#include "mww_verify.h"

namespace mww {

constexpr int kPlaybackMaxSamples = 1 << 22;           // n_samples of a write, min_delay, max_delay and L_ref
constexpr long long kPlaybackMaxStart = 1LL << 50;     // |start| of a write

// x mod C in [0, C), for any sign of x (C > 0)
MWW_HD long long playback_mod(long long x, long long C) {
    const long long r = x % C;
    return r < 0 ? r + C : r;
}

// ---- rows -----------------------------------------------------------------------------------------------------------------------
// Release: at the start of a write call a row whose head w <= S - C is freed.  A heard clip starts at r0 >= S - C >= w, and
// such a row holds only positions before w, so freeing it changes no check.
MWW_HD bool playback_released(long long head, long long seen, int C) { return head <= seen - C; }

// The head a stream without a row starts from when it takes a free row for a write at a: the row counts as holding zeros.
MWW_HD long long playback_fresh_head(long long a, int C) { return a - C; }

// A write of x[0, n) at a into a row of head w: w' = max(w, a + n); positions [span0, a + n) are written, position p with
// p < a (the gap [max(w, w' - C), a) when a > w) as zero, every other as x[p - a]; every other held position keeps its value.
// span0 = max(a, w' - C) when a <= w; len is 0 when the whole write lies before the ring, a + n <= w' - C.
struct PlaybackWrite {
    long long head;     // w'
    long long span0;
    long long len;      // positions [span0, span0 + len)
};
MWW_HD PlaybackWrite playback_write_plan(long long a, int n, long long w, int C) {
    PlaybackWrite p;
    const long long end = a + n;
    p.head = w > end ? w : end;
    const long long lo = p.head - C;
    const long long from = a > w ? w : a;
    p.span0 = from > lo ? from : lo;
    p.len = end > p.span0 ? end - p.span0 : 0;
    return p;
}
// position p of the span: its value
MWW_HD int16_t playback_write_value(const int16_t *x, long long a, long long p) { return p < a ? (int16_t)0 : x[p - a]; }
// 8-sample units when every unit starts on a multiple of 8 in the ring (span0 % 8 == 0, C % 8 == 0) and in the caller's row,
// and is all zeros or all samples (a % 8 == 0, so n % 8 == 0 too); the launcher adds the 16-byte alignment of the caller's audio
MWW_HD bool playback_write_vec_shape(const PlaybackWrite &p, long long a, int n, long long audio_stride) {
    return playback_mod(p.span0, 8) == 0 && playback_mod(a, 8) == 0 && n % 8 == 0 && audio_stride % 8 == 0;
}

// Read: position p of a row of head w (has_row false: a stream without a row) is the ring's slot p mod C when w - C <= p < w,
// else 0.
MWW_HD bool playback_held(long long p, long long head, int C) { return p >= head - C && p < head; }
MWW_HD int16_t playback_read_one(const int16_t *row, int C, bool has_row, long long head, long long p) {
    return has_row && playback_held(p, head, C) ? row[playback_mod(p, C)] : (int16_t)0;
}

// ---- checks ---------------------------------------------------------------------------------------------------------------------
// The reference clip of a slot ending at e: [r1 - L_ref, r1) with r1 = e - min_delay.
MWW_HD long long playback_ref_end(long long e, long long min_delay) { return e - min_delay; }

// Heard: an id in [0, n_streams) whose stream holds a row that still holds the whole clip and whose clip starts before the head:
// r0 >= S - C, r0 >= w - C and r0 < w.
MWW_HD bool playback_heard(int32_t id, int n_streams, bool has_row, long long head, long long r0, long long seen, int C) {
    return id >= 0 && id < n_streams && has_row && r0 >= seen - C && r0 >= head - C && r0 < head;
}

// A slot of a check: sid the stream id that passes when the slot is not flagged, end its clip end e (-1 for no stream).
struct PlaybackSlot { int32_t sid; long long end; };
// mww_playback_check_streams: d_ids[i] ending at d_ends[i]
MWW_HD PlaybackSlot playback_slot_streams(int32_t id, long long end) { return PlaybackSlot{id, end}; }
// mww_playback_check_detections_at: event slot i of a timed detector under mww_verify_detections_at's slot rule: the event's
// stream (verify_slot_id) and e = min(P + post, S)
MWW_HD PlaybackSlot playback_slot_detector(int i, long long count, int capacity, const mww_event *events, const long long *positions, int model,
                                           long long post, long long seen) {
    PlaybackSlot s{verify_slot_id(i, count, capacity, events, model), -1};
    if (s.sid < 0) return s;
    const long long p = positions[i] + post;
    s.end = p < seen ? p : seen;
    return s;
}

// Decision: a heard slot keeps its score and is flagged when (double)score > cutoff (NaN never is); passed is -1 when flagged,
// else the confirmed id.  An unheard slot: NaN, 0, the confirmed id.
struct PlaybackOut { float score; int32_t flagged, passed; };
MWW_HD PlaybackOut playback_decide(bool heard, float score, double cutoff, int32_t confirmed_id) {
    if (!heard) return PlaybackOut{__builtin_nanf(""), 0, confirmed_id};
    const bool f = (double)score > cutoff;
    return PlaybackOut{score, f ? 1 : 0, f ? -1 : confirmed_id};
}

// ---- the host's plan of a write call ------------------------------------------------------------------------------------------
// One entry of a write call's list, staged by the host: stream `stream` takes or keeps row `row` and writes at `start` into a
// row of head `head` (the fresh head for a new row); row -1: the stream's row was released or reset, and its map entry is
// cleared.
struct PlaybackJob { int32_t stream, row; long long start, head; };

// The jobs of a write call from the host's mirror: row_of [n_streams] (-1: none), stream_of [rows] (-1: free) and head [rows];
// listed [n_streams] marks the call's ids.  jobs [0, n) are the writes in list order: a stream keeps its row unless that row
// is released, else it takes the lowest free row (free or released) with the fresh head.  Then one job per released row whose
// stream is not written.  Returns the number of jobs, or -1 when the writes need more rows than are free after the release;
// the mirror is not changed.
inline int playback_plan(const int32_t *ids, const long long *starts, int n, long long seen, int C, int rows, const int32_t *row_of,
                         const int32_t *stream_of, const long long *head, const char *listed, PlaybackJob *jobs) {
    auto released = [&](int r) { return stream_of[r] >= 0 && playback_released(head[r], seen, C); };
    int next = 0, n_jobs = n;
    for (int i = 0; i < n; ++i) {
        int r = row_of[ids[i]];
        if (r >= 0 && !released(r)) {
            jobs[i] = PlaybackJob{ids[i], r, starts[i], head[r]};
            continue;
        }
        while (next < rows && stream_of[next] >= 0 && !released(next)) ++next;
        if (next >= rows) return -1;
        jobs[i] = PlaybackJob{ids[i], next++, starts[i], playback_fresh_head(starts[i], C)};
    }
    for (int r = 0; r < rows; ++r)
        if (released(r) && !listed[stream_of[r]]) jobs[n_jobs++] = PlaybackJob{stream_of[r], -1, 0, 0};
    return n_jobs;
}

// The mirror after a call's jobs: the released rows are freed first (one may be taken again by the call), then every write
// sets its stream's row and the row's head.
inline void playback_commit(const PlaybackJob *jobs, int n, int n_samples, long long seen, int C, int rows, int32_t *row_of, int32_t *stream_of,
                            long long *head) {
    for (int r = 0; r < rows; ++r)
        if (stream_of[r] >= 0 && playback_released(head[r], seen, C)) { row_of[stream_of[r]] = -1; stream_of[r] = -1; }
    for (int i = 0; i < n; ++i) {
        row_of[jobs[i].stream] = jobs[i].row;
        stream_of[jobs[i].row] = jobs[i].stream;
        head[jobs[i].row] = playback_write_plan(jobs[i].start, n_samples, jobs[i].head, C).head;
    }
}

}  // namespace mww
