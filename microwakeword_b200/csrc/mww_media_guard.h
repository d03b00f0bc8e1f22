// mww_media_guard.h -- the bodies of the media guard (include/mww.h, "media guard"): which slots a check hears, the
// fingerprint word of two feature rows, the mismatch test at one lag, the household and time-window filters, and the decision
// of a slot.  The kernels are in mww_media_guard.cu; the history read, reset and features are the existing paths, run through
// their public calls (mww_media_guard_capi.cu).
//
// CUDA-free apart from MWW_HD, so that tests/emul_media_guard.cc runs the same functions on the CPU.
#pragma once

#include <stdint.h>

#include "../../include/mww.h"
#include "mww_common.h"
#include "mww_event_positions.h"
#include "mww_verify.h"

namespace mww {

constexpr int kMediaBits = 39;          // bits per fingerprint word: channel pairs (c, c + 1), c in [0, 39)
constexpr int kMediaMaxLag = 64;
constexpr int kMediaLagChunk = 64;      // the lags of one registered-clip task of the match kernel
constexpr int kMediaMaxSamples = 160000;                       // the longest clip of a rule (n_samples)
constexpr int kMediaMaxWords = (kMediaMaxSamples - 480) / 160;  // its fingerprint words, T - 1

// ---- slots ----------------------------------------------------------------------------------------------------------------------
// One slot of a check: sid is the slot's stream id (passed when the slot is not flagged), rid the id its clip is read from (-1:
// the slot is invalid, read as zeros and never matched), end its clip's end e, pos its position P on the history axis and hh its
// household.
struct MediaSlot { int32_t sid, rid, hh; long long end, pos; };

// The clip [e - n_samples, e) is heard only while all of it is in the ring: e - n_samples >= S - C.
MWW_HD bool media_clip_in_ring(long long end, int n_samples, long long seen, int C) { return end - n_samples >= seen - C; }

// mww_media_check_streams: d_ids[i], ending at d_ends[i], P = e, household d_households[i] (-1 when none are given)
MWW_HD MediaSlot media_slot_streams(int32_t id, long long end, int32_t hh, int n_streams, long long seen, int C, int n_samples) {
    MediaSlot s{id, -1, hh, end, end};
    if (id >= 0 && id < n_streams && media_clip_in_ring(end, n_samples, seen, C)) s.rid = id;
    return s;
}

// mww_media_check_detections_at: event slot i of a timed detector, the verifier's slot rule (verify_slot_id, verify_slot_at),
// P the event's position and the household its group (ev_group nullptr: an ungrouped detector, -1)
MWW_HD MediaSlot media_slot_detector(int i, long long count, int capacity, const mww_event *events, const long long *positions,
                                     const int32_t *ev_group, int model, long long post, long long seen, int C, int n_samples) {
    MediaSlot s{verify_slot_id(i, count, capacity, events, model), -1, -1, -1, -1};
    if (s.sid < 0) return s;
    const SlotAt a = verify_slot_at(i, count, capacity, events, positions, model, post, seen, C, n_samples);
    s.pos = positions[i];
    s.hh = ev_group ? ev_group[i] : -1;
    s.rid = a.id;
    s.end = a.end;
    return s;
}

// ---- fingerprints ---------------------------------------------------------------------------------------------------------------
// Word t - 1 of a clip from its feature rows F[t - 1] (prev) and F[t] (cur): bit c is the sign of the energy difference across
// channels c, c + 1 and frames t - 1, t (Haitsma-Kalker); bits 39..63 are zero.
MWW_HD uint64_t media_fp_word(const uint16_t *prev, const uint16_t *cur) {
    uint64_t w = 0;
    for (int c = 0; c < kMediaBits; ++c) {
        const int32_t d = ((int32_t)cur[c] - (int32_t)cur[c + 1]) - ((int32_t)prev[c] - (int32_t)prev[c + 1]);
        w |= (uint64_t)(d > 0) << c;
    }
    return w;
}

// ---- matching -------------------------------------------------------------------------------------------------------------------
MWW_HD int media_popc(uint64_t x) {
#ifdef __CUDA_ARCH__
    return __popcll(x);
#else
    return __builtin_popcountll(x);
#endif
}

// The overlap of x (n_x words) and y (n_y words) at lag l: t in [t0, t0 + O) with 0 <= t < n_x and 0 <= t + l < n_y.
struct MediaOverlap { int t0, O; };
MWW_HD MediaOverlap media_overlap(int n_x, int n_y, int l) {
    const int a = l < 0 ? -l : 0;
    const int b = n_x < n_y - l ? n_x : n_y - l;
    return MediaOverlap{a, b > a ? b - a : 0};
}

// m mismatches over O words pass when m 1000 <= max_ber_milli 39 O (exact integers)
MWW_HD bool media_ber_passes(long long m, long long O, int max_ber_milli) { return m * 1000 <= (long long)max_ber_milli * kMediaBits * O; }

// Whether x and y match at lag l: O(l) >= min_overlap and the mismatches pass.  y_base: ys holds y[y_base, ...), the words the
// overlap reads.  The sum stops once it has failed (m only grows), which changes no result.
MWW_HD bool media_lag_matches(const uint64_t *x, int n_x, const uint64_t *ys, int y_base, int n_y, int l, int min_overlap, int max_ber_milli) {
    const MediaOverlap o = media_overlap(n_x, n_y, l);
    if (o.O < min_overlap) return false;
    const long long limit = (long long)max_ber_milli * kMediaBits * o.O;
    long long m = 0;
    const uint64_t *y = ys + (l - y_base);
    for (int t = o.t0; t < o.t0 + o.O; ++t) {
        m += media_popc(x[t] ^ y[t]);
        if (m * 1000 > limit) return false;
    }
    return true;
}

// The lags of a pair: [-max_lag, max_lag] between two detections, and every lag with O(l) >= min_overlap against a registered
// clip of n_y words, [-(n_x - min_overlap), n_y - min_overlap].
MWW_HD int media_lag_lo(int n_x, int min_overlap) { return -(n_x - min_overlap); }
MWW_HD int media_lag_hi(int n_y, int min_overlap) { return n_y - min_overlap; }
// registered-clip tasks of the match kernel: kMediaLagChunk lags each
MWW_HD int media_clip_tasks(int n_x, int n_y, int min_overlap) {
    const int lags = media_lag_hi(n_y, min_overlap) - media_lag_lo(n_x, min_overlap) + 1;
    return lags > 0 ? (lags + kMediaLagChunk - 1) / kMediaLagChunk : 0;
}

// Candidate j is heard against slot i: another household, and within window_samples on the history axis.  Same household:
// h_i == h_j >= 0, or h_i == h_j == -1 on one stream.
MWW_HD bool media_same_household(int32_t h_i, int32_t s_i, int32_t h_j, int32_t s_j) { return h_i == h_j && (h_i >= 0 || s_i == s_j); }
MWW_HD bool media_candidate(int32_t h_i, int32_t s_i, long long p_i, int32_t h_j, int32_t s_j, long long p_j, long long window_samples) {
    const long long d = p_j - p_i;
    return !media_same_household(h_i, s_i, h_j, s_j) && (d < 0 ? -d : d) <= window_samples;
}

// ---- decision -------------------------------------------------------------------------------------------------------------------
// A valid slot: matches = its count, media = bit 0 (a registered clip matched) | bit 1 (matches >= min_matches), passed = -1
// when media != 0, else its confirmed id (d_confirmed[i], or sid without d_confirmed).  An invalid slot: -1, 0, confirmed id.
struct MediaOut { int32_t matches, media, passed; };
MWW_HD MediaOut media_decide(bool valid, int32_t count, int32_t clip_hit, int min_matches, int32_t confirmed_id) {
    if (!valid) return MediaOut{-1, 0, confirmed_id};
    const int32_t media = (clip_hit ? 1 : 0) | (count >= min_matches ? 2 : 0);
    return MediaOut{count, media, media ? -1 : confirmed_id};
}

// The ring after a check with `total` valid slots, `count` slots appended before it: valid slot of rank r (its place among
// the call's valid slots) goes to entry (count + r) mod ring, and is written only when r >= total - ring, so that with
// more valid slots than entries the oldest of them are the ones overwritten, and no two slots write one entry.
MWW_HD long long media_ring_entry(long long count, long long total, long long r, int ring) {
    if (ring <= 0 || r < total - ring) return -1;
    return (count + r) % ring;
}

// the device state of a guard's ring: `count` entries appended since the last clear; `base` and `total` the count before the
// current check and its number of valid slots
struct MediaRingState { long long count, base, total; };

}  // namespace mww
