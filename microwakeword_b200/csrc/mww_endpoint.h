// mww_endpoint.h -- the endpointer (mww_endpointer_*, rule in include/mww.h, "endpointing"): the per-row bodies of its four
// kernels (mww_endpoint.cu), the arm replay, the position of a step on the audio history's axis and the index math of the
// command read.  The VAD average is the detectors' own (detector_window_mean, det_add, det_div of mww_detector.h), so a
// row's speech flag is a models detector's VAD `active` bit for bit.
//
// CUDA-free apart from MWW_HD and the two atomics below, so that tests/emul_endpoint.cc runs the same functions on the CPU,
// one row or id at a time as the kernels' threads run them.
#pragma once

#include <stdint.h>

#include "../../include/mww.h"
#include "mww_common.h"
#include "mww_detector.h"
#include "mww_history.h"

namespace mww {

constexpr int kEndpointMaxLookback = 64;     // one uint64 of flags per row

// ---- time axis ----------------------------------------------------------------------------------------------------------------
// The frontend emits a row when it holds 480 samples and then drops hop of them, so after any call it holds the last
// 480 - hop samples of the newest row's window and the b samples that came after it: buffered = (480 - hop) + b, and the
// newest row's window ends at history sample S - b.  Model k's newest step ends g rows (its pending rows) before that, and
// each earlier step s rows before the next.
MWW_HD long long endpoint_position(long long S, int buffered, int hop, int pending, int stride, int n, int j) {
    const long long b = (long long)buffered - (kWindow - hop);
    return S - b - (long long)hop * (pending + (long long)(n - 1 - j) * stride);
}

// Rows the handle emitted between two updates, from the counters read after each: ((S - b) - (S' - b')) / hop.  The update
// fits when that is a whole number R >= 0 and the model's n steps consumed exactly its rows: n s = g' + R - g.
MWW_HD bool endpoint_update_fits(long long S0, int buffered0, int pending0, long long S, int buffered, int pending, int hop, int stride,
                                 int n) {
    const long long moved = (S - buffered) - (S0 - buffered0);
    if (moved < 0 || moved % hop != 0 || n < 0 || pending < 0 || pending >= stride) return false;
    return (long long)n * stride == pending0 + moved / hop - pending;
}

// ---- per-row state (struct-of-arrays, as DetectorArgs) --------------------------------------------------------------------------
struct EndpointArgs {
    mww_endpoint_rule rule;
    int n_rows = 0, n_streams = 0, capacity = 0;
    long long step_samples = 0;                // stride * hop: the samples between two steps
    float *hist = nullptr;                     // [window - 1][n_rows]
    long long *seen = nullptr;                 // [n_rows] steps since the row's last reset
    unsigned long long *flags = nullptr;       // [n_rows] bit i: the flag i steps before the newest
    int32_t *armed = nullptr;                  // [n_rows] the row's global id while armed, else -1
    int32_t *elapsed = nullptr, *run = nullptr, *silence = nullptr, *heard = nullptr;     // [n_rows]
    long long *start = nullptr, *speech_end = nullptr;                                    // [n_rows]
    int32_t *arm_tag = nullptr;                // [n_rows] the last arm call that took the row (one take per call)
    const int32_t *row_of = nullptr;           // [n_streams] global id -> row, -1 for a non-member
    unsigned long long *count = nullptr;
    mww_endpoint_event *events = nullptr;      // [capacity]
    int32_t *ended = nullptr;                  // [capacity]
};

// the last positions of the arm replay: pos[i] is the position of the step i steps before the newest
struct EndpointReplay {
    int steps;                                 // min(lookback_steps, steps consumed since create or the last whole reset)
    int tag;                                   // this arm call
    long long pos[kEndpointMaxLookback];
};

MWW_HD unsigned long long endpoint_claim(unsigned long long *count) {
#if defined(__CUDA_ARCH__)
    return atomicAdd(count, 1ull);
#else
    return (*count)++;
#endif
}
MWW_HD int endpoint_take(int32_t *tag, int value) {
#if defined(__CUDA_ARCH__)
    return atomicExch(tag, value);
#else
    const int old = *tag;
    *tag = value;
    return old;
#endif
}

// ---- speech flag ----------------------------------------------------------------------------------------------------------------
// one row's window - 1 previous probabilities, oldest first, entry j at hist[j * n_rows + r]
struct EndpointHist {
    float *h; int n_rows, r;
    MWW_HD float get(int j) const { return h[(long long)j * n_rows + r]; }
    MWW_HD void set(int j, float v) const { h[(long long)j * n_rows + r] = v; }
};
struct EndpointWindow {
    const EndpointHist &h; int w; float p;
    MWW_HD float operator()(int i) const { return i < w - 1 ? h.get(i) : p; }
};

// The VAD rule of the models detector on probability p: speech = seen >= window && (double)avg > cutoff, `seen` counting
// this step (the caller passes the count before it).  The history moves on by one.
MWW_HD bool endpoint_speech(const EndpointHist &hist, int w, double cutoff, long long seen_before, float p) {
    const float avg = detector_window_mean(EndpointWindow{hist, w, p}, w - 1, w);
    for (int j = 0; j + 1 < w - 1; ++j) hist.set(j, hist.get(j + 1));
    if (w > 1) hist.set(w - 2, p);
    return seen_before + 1 >= w && (double)avg > cutoff;
}

// ---- segmenter ------------------------------------------------------------------------------------------------------------------
struct EndpointSeg {
    int elapsed, run, silence, heard;
    long long start, speech_end;
};
MWW_HD EndpointSeg endpoint_fresh_seg() { return EndpointSeg{0, 0, 0, 0, 0, 0}; }

// one step with flag f at position p, start_sample already placed.  -> the end reason, 0 while the row goes on.  Ties on one
// step go to the first condition that holds.
MWW_HD int endpoint_segment_step(const mww_endpoint_rule &r, EndpointSeg &g, bool f, long long p) {
    g.elapsed += 1;
    if (f) {
        g.run += 1;
        g.silence = 0;
        if (g.run >= r.speech_steps) g.heard = 1;
        if (g.heard) g.speech_end = p;
    } else {
        g.run = 0;
        g.silence += 1;
    }
    if (g.heard && g.silence >= r.silence_steps) return MWW_ENDPOINT_END_OF_SPEECH;
    if (!g.heard && g.elapsed >= r.timeout_steps) return MWW_ENDPOINT_NO_SPEECH;
    if (g.elapsed >= r.max_steps) return MWW_ENDPOINT_MAX_LENGTH;
    return 0;
}
// one step with flag f at position p; the first step after arming places start_sample
MWW_HD int endpoint_segment(const mww_endpoint_rule &r, long long step_samples, EndpointSeg &g, bool f, long long p) {
    if (g.elapsed == 0) g.start = g.speech_end = p - step_samples;
    return endpoint_segment_step(r, g, f, p);
}

MWW_HD EndpointSeg endpoint_load_seg(const EndpointArgs &a, int r) {
    return EndpointSeg{a.elapsed[r], a.run[r], a.silence[r], a.heard[r], a.start[r], a.speech_end[r]};
}
MWW_HD void endpoint_store_seg(const EndpointArgs &a, int r, const EndpointSeg &g) {
    a.elapsed[r] = g.elapsed; a.run[r] = g.run; a.silence[r] = g.silence; a.heard[r] = g.heard;
    a.start[r] = g.start; a.speech_end[r] = g.speech_end;
}

// the event of a row that ended on the step at position p: a slot through the counter, the id into `ended` beside it
MWW_HD void endpoint_emit(const EndpointArgs &a, int32_t id, int reason, const EndpointSeg &g, long long p) {
    const unsigned long long slot = endpoint_claim(a.count);
    if (slot >= (unsigned long long)a.capacity) return;
    mww_endpoint_event e;
    e.stream = id; e.reason = reason; e.start_sample = g.start; e.end_sample = p; e.speech_end_sample = g.speech_end;
    e.steps = g.elapsed; e.pad = 0;
    a.events[slot] = e;
    a.ended[slot] = id;
}

// ---- the four kernels' bodies ---------------------------------------------------------------------------------------------------
// The positioned forms (kAt, libmww_endpoint_at.so; include/mww.h, "positioned arm") also keep each row's mute word,
// mute[r]: the low bits count the update steps that still take flag 0, and kEndpointPlaced marks a row whose start_sample
// an arm_at fixed and which has taken no step since.  Every form that gives a row fresh segmenter state sets the word to 0.
// The plain forms (kAt = false) neither read nor write it.
constexpr int32_t kEndpointPlaced = 1 << 30;
constexpr int32_t kEndpointMuteSteps = kEndpointPlaced - 1;

// update, row r: n steps of probs[r * pitch + j], step j at position pos0 + j * step_samples, in order.  Every row takes the
// flag; an armed row then runs the segmenter, and disarms when it ends.  A row that is not armed keeps fresh segmenter state.
template <bool kAt>
MWW_HD void endpoint_update_row_t(const EndpointArgs &a, int32_t *mute, int r, const float *probs, long long pitch, int n, long long pos0) {
    const EndpointHist hist{a.hist, a.n_rows, r};
    const int w = a.rule.vad_window;
    long long seen = a.seen[r];
    unsigned long long flags = a.flags[r];
    int32_t id = a.armed[r];
    const bool was_armed = id >= 0;
    EndpointSeg g = was_armed ? endpoint_load_seg(a, r) : endpoint_fresh_seg();
    int32_t m = 0;
    if constexpr (kAt) m = was_armed ? mute[r] : 0;
    const float *row = probs + (long long)r * pitch;
    for (int j = 0; j < n; ++j) {
        const bool f = endpoint_speech(hist, w, a.rule.vad_cutoff, seen, row[j]);
        seen += 1;
        flags = flags << 1 | (f ? 1ull : 0ull);
        if (id < 0) continue;
        const long long p = pos0 + (long long)j * a.step_samples;
        int reason;
        if constexpr (kAt) {
            // a muted step takes flag 0 (the stored flag keeps f); a placed row's first step leaves start_sample where it is
            const bool muted = (m & kEndpointMuteSteps) != 0;
            const bool placed = (m & kEndpointPlaced) != 0;
            m = (m & kEndpointMuteSteps) - (muted ? 1 : 0);
            reason = placed ? endpoint_segment_step(a.rule, g, f && !muted, p) : endpoint_segment(a.rule, a.step_samples, g, f && !muted, p);
        } else {
            reason = endpoint_segment(a.rule, a.step_samples, g, f, p);
        }
        if (reason) {
            endpoint_emit(a, id, reason, g, p);
            id = -1;
            g = endpoint_fresh_seg();
            m = 0;
        }
    }
    a.seen[r] = seen;
    a.flags[r] = flags;
    if (was_armed) {
        a.armed[r] = id;
        endpoint_store_seg(a, r, g);
        if constexpr (kAt) mute[r] = m;
    }
}
MWW_HD void endpoint_update_row(const EndpointArgs &a, int r, const float *probs, long long pitch, int n, long long pos0) {
    endpoint_update_row_t<false>(a, nullptr, r, probs, pitch, n, pos0);
}

// arm, one listed global id: a member row not yet taken by this call gets fresh segmenter state and replays its last
// R.steps flags, oldest first, at their positions.  Ids outside the set (-1 included) are ignored.
template <bool kAt>
MWW_HD void endpoint_arm_one_t(const EndpointArgs &a, int32_t *mute, const EndpointReplay &R, int32_t id) {
    if (id < 0 || id >= a.n_streams) return;
    const int r = a.row_of[id];
    if (r < 0 || endpoint_take(&a.arm_tag[r], R.tag) == R.tag) return;
    EndpointSeg g = endpoint_fresh_seg();
    const unsigned long long flags = a.flags[r];
    int32_t armed = id;
    for (int i = R.steps - 1; i >= 0; --i) {
        const long long p = R.pos[i];
        if (const int reason = endpoint_segment(a.rule, a.step_samples, g, (flags >> i) & 1ull, p)) {
            endpoint_emit(a, id, reason, g, p);
            armed = -1;
            g = endpoint_fresh_seg();
            break;
        }
    }
    a.armed[r] = armed;
    endpoint_store_seg(a, r, g);
    if constexpr (kAt) mute[r] = 0;
}
MWW_HD void endpoint_arm_one(const EndpointArgs &a, const EndpointReplay &R, int32_t id) { endpoint_arm_one_t<false>(a, nullptr, R, id); }

// disarm (reset = 0) or reset (reset = 1) of row r: disarming drops the segment without an event; a reset also gives fresh
// VAD state (zero history, seen 0, every flag 0)
template <bool kAt>
MWW_HD void endpoint_clear_row_t(const EndpointArgs &a, int32_t *mute, int r, int reset) {
    a.armed[r] = -1;
    endpoint_store_seg(a, r, endpoint_fresh_seg());
    if constexpr (kAt) mute[r] = 0;
    if (!reset) return;
    for (int j = 0; j < a.rule.vad_window - 1; ++j) a.hist[(long long)j * a.n_rows + r] = 0.0f;
    a.seen[r] = 0;
    a.flags[r] = 0;
}
MWW_HD void endpoint_clear_row(const EndpointArgs &a, int r, int reset) { endpoint_clear_row_t<false>(a, nullptr, r, reset); }
// the row of a listed global id, -1 for an id outside the set
MWW_HD int endpoint_row(const EndpointArgs &a, int32_t id) { return id >= 0 && id < a.n_streams ? a.row_of[id] : -1; }

// ---- positioned arm (mww_endpointer_arm_at): two launches, a reduction of each row's latest position, then the arm --------------
// what both passes take beside EndpointArgs: the replay of arm, q (the position of the newest step consumed: endpoint_position
// of the baseline with n = 1), the skip in samples, the rows' mute words and the reduction's keys
struct EndpointAt {
    EndpointReplay R;
    long long q, skip;
    int32_t *mute;
    unsigned long long *key;               // [n_rows] the latest P' of the call as an ordered key; 0 (none) between calls
};
// a position as an unsigned key in the same order, 0 for the smallest
MWW_HD unsigned long long endpoint_at_key(long long P) { return (unsigned long long)P ^ 0x8000000000000000ull; }
MWW_HD long long endpoint_at_clamp(long long P, long long q) { return P < q ? P : q; }

// pass 1, one listed (id, P): the row's key becomes the largest P' = min(P, q) listed for it
MWW_HD void endpoint_at_reduce_one(const EndpointArgs &a, const EndpointAt &A, int32_t id, long long P) {
    const int r = endpoint_row(a, id);
    if (r < 0) return;
    const unsigned long long k = endpoint_at_key(endpoint_at_clamp(P, A.q));
#if defined(__CUDA_ARCH__)
    atomicMax(&A.key[r], k);
#else
    if (k > A.key[r]) A.key[r] = k;
#endif
}

// pass 2, one listed (id, P): the slot whose P' is the row's latest takes the row (one take per call; equal positions arm
// alike) and puts its key back to 0.  The row gets fresh segmenter state with start_sample = speech_end_sample = P', replays the
// steps of R after P', each with flag f && p > P' + skip, and keeps the mute word of the steps still within the skip.  A slot
// that reads the key after the taker cleared it reads 0, the key of no position a later slot could still take with.
MWW_HD void endpoint_arm_at_one(const EndpointArgs &a, const EndpointAt &A, int32_t id, long long P) {
    const int r = endpoint_row(a, id);
    if (r < 0) return;
    const long long Pc = endpoint_at_clamp(P, A.q);
    if (endpoint_at_key(Pc) != A.key[r] || endpoint_take(&a.arm_tag[r], A.R.tag) == A.R.tag) return;
    A.key[r] = 0;
    EndpointSeg g = endpoint_fresh_seg();
    g.start = g.speech_end = Pc;
    const unsigned long long flags = a.flags[r];
    int32_t armed = id;
    for (int i = A.R.steps - 1; i >= 0; --i) {
        const long long p = A.R.pos[i];
        if (p <= Pc) continue;
        if (const int reason = endpoint_segment_step(a.rule, g, ((flags >> i) & 1ull) && p > Pc + A.skip, p)) {
            endpoint_emit(a, id, reason, g, p);
            armed = -1;
            g = endpoint_fresh_seg();
            break;
        }
    }
    int32_t m = 0;
    if (armed >= 0) {
        const long long d = Pc + A.skip - A.q;                  // future steps q + k stride hop with k >= 1 that are <= P' + skip
        m = d > 0 ? (int32_t)(d / a.step_samples) : 0;
        if (g.elapsed == 0) m |= kEndpointPlaced;
    }
    a.armed[r] = armed;
    endpoint_store_seg(a, r, g);
    A.mute[r] = m;
}

// ---- command read ---------------------------------------------------------------------------------------------------------------
// event slot i's samples [a, a + len) on the history axis: a = start - pre; the end is min(speech_end + post, end) for
// END_OF_SPEECH and end otherwise; len is capped at max_samples, keeping the beginning.  An unused slot has len 0.
struct CommandSpan { long long a; int len; };
MWW_HD CommandSpan endpoint_command_span(int i, long long count, int capacity, const mww_endpoint_event *events, long long pre, long long post,
                                         int max_samples) {
    CommandSpan c{0, 0};
    if ((long long)i >= (count < (long long)capacity ? count : (long long)capacity)) return c;
    const mww_endpoint_event e = events[i];
    long long end = e.end_sample;
    if (e.reason == MWW_ENDPOINT_END_OF_SPEECH && e.speech_end_sample + post < end) end = e.speech_end_sample + post;
    c.a = e.start_sample - pre;
    const long long len = end - c.a;
    c.len = len <= 0 ? 0 : (len < max_samples ? (int)len : max_samples);
    return c;
}
// history sample t of stream id, `seen` samples appended: zero outside [seen - C, seen), where the ring holds other samples
// or none yet (entries from before a reset are zeros in the ring itself)
MWW_HD bool endpoint_in_ring(long long t, long long seen, int C) { return t >= seen - C && t < seen; }
MWW_HD int16_t endpoint_command_one(const int16_t *ring, int C, long long seen, int id, long long t) {
    return endpoint_in_ring(t, seen, C) ? ring[(long long)id * C + history_mod(t, C)] : (int16_t)0;
}

}  // namespace mww
