// emul_media_guard.cc -- the bodies of the media guard (microwakeword_b200/csrc/mww_media_guard.h) on the CPU, for
// tests/test_media_guard.py: fingerprints of feature rows as media_fingerprint_kernel makes them, a slot of each form, and one
// check as the match and decide kernels run it -- every (slot, candidate) pair through the filters and the lag tests, the
// registered clips in lag chunks, then the decision and the ring append by rank.
#include <vector>

#include "../microwakeword_b200/csrc/mww_media_guard.h"

using namespace mww;

extern "C" {

int emul_sizes(int *rule, int *desc) {
    *rule = (int)sizeof(mww_media_rule);
    *desc = (int)sizeof(mww_media_guard_desc);
    return 0;
}

void emul_fingerprint(const uint16_t *feat, int n, int rows, int words, uint64_t *fp) {
    for (int s = 0; s < n; ++s)
        for (int t = 0; t < words; ++t) {
            const uint16_t *r = feat + ((long long)s * rows + t) * kNumChannels;
            fp[(long long)s * words + t] = media_fp_word(r, r + kNumChannels);
        }
}

// media_slot_streams of n ids: rid and valid flag per slot
void emul_slots_streams(int n, const int32_t *ids, const long long *ends, int n_streams, long long seen, int C, int n_samples, int32_t *rid) {
    for (int i = 0; i < n; ++i) rid[i] = media_slot_streams(ids[i], ends[i], -1, n_streams, seen, C, n_samples).rid;
}

// media_slot_detector of every event slot [0, capacity) of a timed detector (ev_group nullptr: ungrouped)
void emul_slots_detector(int capacity, long long count, const mww_event *events, const long long *positions, const int32_t *ev_group, int model,
                         long long post, long long seen, int C, int n_samples, int32_t *sid, int32_t *rid, int32_t *hh, long long *end,
                         long long *pos) {
    for (int i = 0; i < capacity; ++i) {
        const MediaSlot s = media_slot_detector(i, count, capacity, events, positions, ev_group, model, post, seen, C, n_samples);
        sid[i] = s.sid; rid[i] = s.rid; hh[i] = s.hh; end[i] = s.end; pos[i] = s.pos;
    }
}

// One check of n slots (fingerprints fp [n][W], rid -1 for an invalid slot, sid, hh, pos), a ring of `ring` entries with
// `*count` appended so far, and n_clips registered clips (clip_fp back to back, clip_len words each).  Writes matches, media,
// passed and the ring, and advances *count.
void emul_check(int n, int W, const uint64_t *fp, const int32_t *sid, const int32_t *rid, const int32_t *hh, const long long *pos,
                const int32_t *confirmed, int ring, long long *count, uint64_t *ring_fp, int32_t *ring_stream, int32_t *ring_hh,
                long long *ring_pos, int n_clips, const uint64_t *clip_fp, const int32_t *clip_len, int max_lag, int min_overlap,
                int max_ber_milli, int min_matches, long long window, int32_t *matches, int32_t *media, int32_t *passed) {
    const long long base = *count, fill = ring > 0 ? (base < ring ? base : ring) : 0;
    std::vector<int32_t> cnt(n, 0), hit(n, 0), rank(n, -1);
    long long total = 0;
    for (int i = 0; i < n; ++i)
        if (rid[i] >= 0) rank[i] = (int32_t)total++;
    for (int i = 0; i < n; ++i) {
        if (rid[i] < 0) continue;
        const uint64_t *x = fp + (long long)i * W;
        auto any_lag = [&](const uint64_t *ys, int y_base, int ny, int lo, int hi) {
            for (int l = lo; l <= hi; ++l)
                if (media_lag_matches(x, W, ys, y_base, ny, l, min_overlap, max_ber_milli)) return true;
            return false;
        };
        for (int j = 0; j < n; ++j)
            if (j != i && rid[j] >= 0 && media_candidate(hh[i], rid[i], pos[i], hh[j], rid[j], pos[j], window) &&
                any_lag(fp + (long long)j * W, 0, W, -max_lag, max_lag))
                ++cnt[i];
        for (long long r = 0; r < fill; ++r)
            if (media_candidate(hh[i], rid[i], pos[i], ring_hh[r], ring_stream[r], ring_pos[r], window) &&
                any_lag(ring_fp + r * W, 0, W, -max_lag, max_lag))
                ++cnt[i];
        long long off = 0;
        for (int k = 0; k < n_clips; ++k) {
            const int ny = clip_len[k], top = media_lag_hi(ny, min_overlap);
            for (int c = 0; c < media_clip_tasks(W, ny, min_overlap); ++c) {
                const int lo = media_lag_lo(W, min_overlap) + c * kMediaLagChunk;
                const int hi = lo + kMediaLagChunk - 1 < top ? lo + kMediaLagChunk - 1 : top;
                const int y_base = lo > 0 ? lo : 0;
                if (any_lag(clip_fp + off + y_base, y_base, ny, lo, hi)) hit[i] = 1;
            }
            off += ny;
        }
    }
    for (int i = 0; i < n; ++i) {
        const MediaOut o = media_decide(rid[i] >= 0, cnt[i], hit[i], min_matches, confirmed ? confirmed[i] : sid[i]);
        matches[i] = o.matches; media[i] = o.media; passed[i] = o.passed;
    }
    for (int i = 0; i < n; ++i) {
        if (rid[i] < 0) continue;
        const long long e = media_ring_entry(base, total, rank[i], ring);
        if (e < 0) continue;
        for (int t = 0; t < W; ++t) ring_fp[e * W + t] = fp[(long long)i * W + t];
        ring_stream[e] = rid[i]; ring_hh[e] = hh[i]; ring_pos[e] = pos[i];
    }
    *count = base + total;
}

}  // extern "C"
