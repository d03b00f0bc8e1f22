// mww_media_guard_capi.cu -- the extern "C" entry points of the media guard (include/mww.h, "media guard").  Host code only:
// the kernels are in mww_media_guard.{h,cu}.  A guard is an object of its own, like a verifier: it reads a source handle and a
// detector through their public calls (and a grouped detector's event groups through detector_event_groups), turns clips into
// feature rows on frontend-only handles of its own through mww_features, and its messages go to mww_last_error(NULL).
#include <cstring>
#include <string>
#include <vector>

#include "mww_capi.h"
#include "mww_kernels.h"

using namespace mww;

struct mww_media_guard {
    int device = 0, slots = 0, frames = 0, words = 0;   // frames T and words W = T - 1 of a slot's clip
    mww_media_rule rule{};
    mww_t *h = nullptr;                 // frontend-only, `slots` streams: the slots' clips, fully reset by every check
    mww_t *hm = nullptr;                // frontend-only, 1 stream: registered clips (max_media > 0)
    int clip_frames = 0;                // T of the longest registrable clip
    long long launches = 0;             // the guard's own kernel launches
    int16_t *d_audio = nullptr;         // [slots][n_samples]
    uint16_t *d_feat = nullptr;         // [slots][T][40]
    uint64_t *d_fp = nullptr;           // [slots][W]
    int32_t *sid = nullptr, *rid = nullptr, *hh = nullptr, *rank = nullptr, *count = nullptr, *clip_hit = nullptr;   // [slots]
    long long *end = nullptr, *pos = nullptr;                                                                       // [slots]
    MediaRingState *state = nullptr;
    uint64_t *ring_fp = nullptr;        // [ring][W]
    int32_t *ring_stream = nullptr, *ring_hh = nullptr;
    long long *ring_pos = nullptr;
    uint16_t *m_feat = nullptr;         // [clip_frames][40]
    uint64_t *clip_fp = nullptr;        // [max_media (clip_frames - 1)], the registered clips back to back
    long long *clip_off = nullptr;      // [max_media]
    int32_t *clip_len = nullptr, *clip_task0 = nullptr;   // [max_media], [max_media + 1]
    std::vector<long long> h_off;       // host copies of the registered clips' offsets, lengths and first match tasks
    std::vector<int32_t> h_len, h_task0;
    int n_clips = 0;
    long long clip_words = 0, clip_tasks = 0;
};

namespace {

constexpr int kMediaMinSamples = 640, kMediaMaxClips = 4096, kMediaMaxClipSamples = 1 << 24;
constexpr long long kMediaMaxRing = 1 << 20, kMediaMaxWindow = 1LL << 40, kMediaMaxClipWords = 1LL << 27, kMediaMaxPost = 1 << 22;

#define GCU(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return cuda_fail(nullptr, e_, #call); } while (0)

int refuse(const std::string &msg) { return fail(nullptr, MWW_EINVAL, msg); }

int pass_on(int rc, const mww_t *h, const std::string &what) {
    const char *m = mww_last_error(h);
    return fail(nullptr, rc, what + ": " + (m ? m : "failed"));
}

int frames_of(int n_samples) { return (n_samples - kWindow) / kHop + 1; }

void guard_free(mww_media_guard_t *g) {
    if (g->h) mww_destroy(g->h);
    if (g->hm) mww_destroy(g->hm);
    cudaFree(g->d_audio); cudaFree(g->d_feat); cudaFree(g->d_fp);
    cudaFree(g->sid); cudaFree(g->rid); cudaFree(g->hh); cudaFree(g->rank); cudaFree(g->count); cudaFree(g->clip_hit);
    cudaFree(g->end); cudaFree(g->pos); cudaFree(g->state);
    cudaFree(g->ring_fp); cudaFree(g->ring_stream); cudaFree(g->ring_hh); cudaFree(g->ring_pos);
    cudaFree(g->m_feat); cudaFree(g->clip_fp); cudaFree(g->clip_off); cudaFree(g->clip_len); cudaFree(g->clip_task0);
    delete g;
}

// Every buffer, and the frontend scratch of both handles: one features call on zeroed audio of the largest size sizes it, so
// that no check or register allocates.
int guard_alloc(mww_media_guard_t *g) {
    const size_t S = (size_t)g->slots, N = (size_t)g->rule.n_samples, T = (size_t)g->frames, W = (size_t)g->words;
    const size_t R = (size_t)g->rule.ring, M = (size_t)g->rule.max_media;
    GCU(cudaMalloc(&g->d_audio, S * N * sizeof(int16_t)));
    GCU(cudaMalloc(&g->d_feat, S * T * kNumChannels * sizeof(uint16_t)));
    GCU(cudaMalloc(&g->d_fp, S * W * sizeof(uint64_t)));
    for (int32_t **p : {&g->sid, &g->rid, &g->hh, &g->rank, &g->count, &g->clip_hit}) GCU(cudaMalloc(p, S * sizeof(int32_t)));
    GCU(cudaMalloc(&g->end, S * sizeof(long long)));
    GCU(cudaMalloc(&g->pos, S * sizeof(long long)));
    GCU(cudaMalloc(&g->state, sizeof(MediaRingState)));
    GCU(cudaMemset(g->state, 0, sizeof(MediaRingState)));
    GCU(cudaMalloc(&g->ring_fp, std::max<size_t>(R * W, 1) * sizeof(uint64_t)));
    GCU(cudaMalloc(&g->ring_stream, std::max<size_t>(R, 1) * sizeof(int32_t)));
    GCU(cudaMalloc(&g->ring_hh, std::max<size_t>(R, 1) * sizeof(int32_t)));
    GCU(cudaMalloc(&g->ring_pos, std::max<size_t>(R, 1) * sizeof(long long)));
    const size_t CW = g->clip_frames > 1 ? (size_t)(g->clip_frames - 1) : 0;
    GCU(cudaMalloc(&g->m_feat, std::max<size_t>((size_t)g->clip_frames * kNumChannels, 1) * sizeof(uint16_t)));
    GCU(cudaMalloc(&g->clip_fp, std::max<size_t>(M * CW, 1) * sizeof(uint64_t)));
    GCU(cudaMalloc(&g->clip_off, std::max<size_t>(M, 1) * sizeof(long long)));
    GCU(cudaMalloc(&g->clip_len, std::max<size_t>(M, 1) * sizeof(int32_t)));
    GCU(cudaMalloc(&g->clip_task0, (M + 1) * sizeof(int32_t)));
    g->h_off.assign(M, 0);
    g->h_len.assign(M, 0);
    g->h_task0.assign(M + 1, 0);
    GCU(cudaMemset(g->d_audio, 0, S * N * sizeof(int16_t)));
    int rows = 0;
    if (int rc = mww_features(g->h, g->d_audio, g->rule.n_samples, g->rule.n_samples, g->d_feat, g->frames, &rows, nullptr))
        return pass_on(rc, g->h, "mww_media_guard_create");
    if (g->hm) {
        int16_t *zeros = nullptr;
        GCU(cudaMalloc(&zeros, (size_t)g->rule.max_media_samples * sizeof(int16_t)));
        cudaMemset(zeros, 0, (size_t)g->rule.max_media_samples * sizeof(int16_t));
        const int rc = mww_features(g->hm, zeros, g->rule.max_media_samples, g->rule.max_media_samples, g->m_feat, g->clip_frames, &rows, nullptr);
        cudaDeviceSynchronize();
        cudaFree(zeros);
        if (rc) return pass_on(rc, g->hm, "mww_media_guard_create");
    }
    GCU(cudaDeviceSynchronize());
    return MWW_OK;
}

// The checks both calls share, before any device work: the guard and src, src's audio history and device, the number of
// slots, and (probe: a read of nothing, which refuses a poisoned handle and launches nothing) src's health.
int check_source(const mww_media_guard_t *g, mww_t *src, const std::string &call, int n, mww_info *info, int *C, long long *S, cudaStream_t st) {
    if (!g || !src) return refuse(call + ": needs a media guard and a source handle");
    if (n < 0 || n > g->slots) return refuse(call + ": " + std::to_string(n) + " slots for a media guard of " + std::to_string(g->slots));
    if (mww_get_info(src, info) != MWW_OK) return refuse(call + ": cannot read the source handle");
    if (info->device != g->device) return refuse(call + ": the source handle is on another device than the media guard");
    mww_get_audio_history(src, C, S);
    if (*C < g->rule.n_samples)
        return refuse(call + ": the source handle keeps " + (*C ? std::to_string(*C) + " samples of audio history" : std::string("no audio history")) +
                      "; the media guard reads " + std::to_string(g->rule.n_samples));
    if (mww_read_audio_history_device_ids(src, nullptr, 0, 0, nullptr, 0, st) != MWW_OK)
        return refuse(call + ": the source handle cannot be read: " + mww_last_error(src));
    return MWW_OK;
}

// The pass over n slots: the slots kernel, src's history read that ends at each slot's clip end, a fresh frontend's rows,
// their fingerprints, the match and the decision with the ring append.  A constant number of launches for n >= 1.
int run(mww_media_guard_t *g, mww_t *src, const MediaSlotsArgs &sa, const int32_t *d_confirmed, int32_t *d_matches, int32_t *d_media,
        int32_t *d_passed, cudaStream_t st, const std::string &call) {
    const int N = g->rule.n_samples, n = sa.n;
    const MediaSlotsOut so{g->sid, g->rid, g->hh, g->rank, g->count, g->clip_hit, g->end, g->pos, g->state};
    GCU(launch_media_slots(sa, so, st));
    if (int rc = mww_read_audio_history_at(src, g->rid, g->end, n, N, g->d_audio, N, st)) return pass_on(rc, src, call + ": history read");
    if (int rc = mww_reset(g->h, nullptr, 0, st)) return pass_on(rc, g->h, call + ": frontend reset");
    int rows = 0;
    if (int rc = mww_features(g->h, g->d_audio, N, N, g->d_feat, g->frames, &rows, st)) return pass_on(rc, g->h, call + ": features");
    GCU(launch_media_fingerprint(g->d_feat, g->frames, n, g->words, g->d_fp, g->words, st));
    MediaMatchArgs ma{};
    ma.fp = g->d_fp; ma.words = g->words; ma.n = n;
    ma.rid = g->rid; ma.hh = g->hh; ma.pos = g->pos;
    ma.ring_fp = g->ring_fp; ma.ring_stream = g->ring_stream; ma.ring_hh = g->ring_hh; ma.ring_pos = g->ring_pos; ma.ring = g->rule.ring;
    ma.state = g->state;
    ma.clip_fp = g->clip_fp; ma.clip_off = g->clip_off; ma.clip_len = g->clip_len; ma.clip_task0 = g->clip_task0;
    ma.n_clips = g->n_clips;
    ma.clip_tasks = g->clip_tasks;
    ma.max_lag = g->rule.max_lag; ma.min_overlap = g->rule.min_overlap; ma.max_ber_milli = g->rule.max_ber_milli; ma.window = g->rule.window_samples;
    ma.count = g->count; ma.clip_hit = g->clip_hit;
    GCU(launch_media_match(ma, st));
    MediaDecideArgs da{};
    da.n = n; da.words = g->words; da.ring = g->rule.ring; da.min_matches = g->rule.min_matches;
    da.fp = g->d_fp; da.sid = g->sid; da.rid = g->rid; da.hh = g->hh; da.rank = g->rank; da.count = g->count; da.clip_hit = g->clip_hit;
    da.confirmed = d_confirmed; da.pos = g->pos; da.state = g->state;
    da.matches = d_matches; da.media = d_media; da.passed = d_passed;
    da.ring_fp = g->ring_fp; da.ring_stream = g->ring_stream; da.ring_hh = g->ring_hh; da.ring_pos = g->ring_pos;
    GCU(launch_media_decide(da, st));
    g->launches += 4;
    return MWW_OK;
}

long long state_bytes(const mww_media_guard_t *g, int n_media, long long media_words) {
    const long long R = g->rule.ring, W = g->words;
    return 32 + R * W * 8 + R * 8 + R * 4 * 2 + (long long)n_media * 8 + media_words * 8;
}

}  // namespace

extern "C" {

int mww_media_guard_create(int device, int slots, const mww_media_rule *rule, mww_media_guard_t **out) {
    const std::string call = "mww_media_guard_create: ";
    if (!out) return refuse(call + "out is NULL");
    *out = nullptr;
    if (!rule) return refuse(call + "rule is NULL");
    const mww_media_rule &r = *rule;
    if (slots < 1) return refuse(call + "slots must be at least 1");
    if (r.n_samples < kMediaMinSamples || r.n_samples > kMediaMaxSamples) return refuse(call + "n_samples must be in [640, 160000]");
    const int W = frames_of(r.n_samples) - 1;
    if (r.max_lag < 0 || r.max_lag > kMediaMaxLag) return refuse(call + "max_lag must be in [0, 64]");
    if (r.min_overlap < 1 || r.min_overlap > W)
        return refuse(call + "min_overlap must be in [1, " + std::to_string(W) + "] (the clip's fingerprint words)");
    if (r.max_lag > W - r.min_overlap) return refuse(call + "max_lag must be at most the clip's words minus min_overlap");
    if (r.max_ber_milli < 0 || r.max_ber_milli > 500) return refuse(call + "max_ber_milli must be in [0, 500]");
    if (r.min_matches < 1) return refuse(call + "min_matches must be at least 1");
    if (r.ring < 0 || r.ring > kMediaMaxRing) return refuse(call + "ring must be in [0, 2^20]");
    if (r.window_samples < 0 || r.window_samples > kMediaMaxWindow) return refuse(call + "window_samples must be in [0, 2^40]");
    if (r.max_media < 0 || r.max_media > kMediaMaxClips) return refuse(call + "max_media must be in [0, 4096]");
    if (r.max_media_samples < 0 || r.max_media_samples > kMediaMaxClipSamples) return refuse(call + "max_media_samples must be in [0, 2^24]");
    int clip_frames = 0;
    if (r.max_media > 0) {
        if (r.max_media_samples < kMediaMinSamples) return refuse(call + "max_media_samples must be at least 640 when max_media > 0");
        clip_frames = frames_of(r.max_media_samples);
        if (clip_frames - 1 < r.min_overlap) return refuse(call + "max_media_samples gives fewer fingerprint words than min_overlap");
        if ((long long)r.max_media * (clip_frames - 1) > kMediaMaxClipWords) return refuse(call + "max_media x the longest clip's words must be at most 2^27");
    }
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0)
        return fail(nullptr, MWW_ECUDA, std::string("no CUDA device available (this library has no CPU fallback): ") + cudaGetErrorString(e));
    mww_media_guard_t *g = new mww_media_guard;
    g->device = device; g->slots = slots; g->frames = W + 1; g->words = W; g->rule = r; g->clip_frames = clip_frames;
    if (int rc = mww_create(nullptr, 0, device, slots, &g->h)) { guard_free(g); return rc; }
    if (r.max_media > 0) {
        if (int rc = mww_create(nullptr, 0, device, 1, &g->hm)) { guard_free(g); return rc; }
    }
    DeviceGuard guard(device);
    if (guard.err != cudaSuccess) { guard_free(g); return cuda_fail(nullptr, guard.err, "cudaSetDevice"); }
    if (int rc = guard_alloc(g)) { guard_free(g); return rc; }
    *out = g;
    return MWW_OK;
}

int mww_media_guard_destroy(mww_media_guard_t *g) {
    if (!g) return MWW_OK;
    DeviceGuard guard(g->device);
    cudaDeviceSynchronize();
    guard_free(g);
    return MWW_OK;
}

int mww_media_guard_info(const mww_media_guard_t *g, mww_media_guard_desc *out) {
    if (!g || !out) return refuse("mww_media_guard_info: needs a media guard and out");
    DeviceGuard guard(g->device);
    if (guard.err != cudaSuccess) return cuda_fail(nullptr, guard.err, "cudaSetDevice");
    MediaRingState s{};
    GCU(cudaDeviceSynchronize());
    GCU(cudaMemcpy(&s, g->state, sizeof(s), cudaMemcpyDeviceToHost));
    *out = mww_media_guard_desc{};
    out->slots = g->slots; out->frames = g->frames; out->device = g->device; out->rule = g->rule;
    out->n_media = g->n_clips;
    out->ring_count = s.count;
    out->ring_fill = std::min<long long>(s.count, g->rule.ring);
    out->launches = g->launches + mww_launch_count(g->h) + (g->hm ? mww_launch_count(g->hm) : 0);
    return MWW_OK;
}

int mww_media_check_streams(mww_media_guard_t *g, mww_t *src, const int32_t *d_ids, const long long *d_ends, const int32_t *d_households, int n,
                            const int32_t *d_confirmed, int32_t *d_matches, int32_t *d_media, int32_t *d_passed, void *cu_stream) {
    const std::string call = "mww_media_check_streams";
    cudaStream_t st = static_cast<cudaStream_t>(cu_stream);
    mww_info info;
    int C = 0;
    long long S = 0;
    if (int rc = check_source(g, src, call, n, &info, &C, &S, st)) return rc;
    if (n > 0 && (!d_ids || !d_ends)) return refuse(call + ": d_ids and d_ends must not be NULL");
    if (n == 0) return MWW_OK;
    DeviceGuard guard(g->device);
    if (guard.err != cudaSuccess) return cuda_fail(nullptr, guard.err, "cudaSetDevice");
    MediaSlotsArgs sa{};
    sa.n = n; sa.n_streams = info.n_streams; sa.C = C; sa.n_samples = g->rule.n_samples; sa.seen = S;
    sa.ids = d_ids; sa.ends = d_ends; sa.households = d_households;
    return run(g, src, sa, d_confirmed, d_matches, d_media, d_passed, st, call);
}

int mww_media_check_detections_at(mww_media_guard_t *g, mww_t *src, mww_detector_t *det, int model, long long post, const int32_t *d_confirmed,
                                  int32_t *d_matches, int32_t *d_media, int32_t *d_passed, void *cu_stream) {
    const std::string call = "mww_media_check_detections_at";
    if (!g) return refuse(call + ": needs a media guard and a source handle");
    if (!det) return refuse(call + ": detector is NULL");
    if (post < 0 || post > kMediaMaxPost) return refuse(call + ": post must be in [0, 2^22]");
    const int64_t *d_positions = nullptr;
    if (mww_get_detector_positions(det, &d_positions) != MWW_OK)
        return refuse(call + ": the detector is not timed (mww_time_detector_events): its events carry no positions");
    const long long *d_count = nullptr;
    const mww_event *d_events = nullptr;
    int capacity = 0;
    mww_detector_buffers(det, &d_count, &d_events, nullptr, &capacity);
    if (capacity > g->slots)
        return refuse(call + ": the detector keeps " + std::to_string(capacity) + " events; the media guard has " + std::to_string(g->slots) + " slots");
    cudaStream_t st = static_cast<cudaStream_t>(cu_stream);
    mww_info info;
    int C = 0;
    long long S = 0;
    if (int rc = check_source(g, src, call, capacity, &info, &C, &S, st)) return rc;
    cudaPointerAttributes attr;
    if (cudaPointerGetAttributes(&attr, d_count) != cudaSuccess || attr.device != g->device) {
        cudaGetLastError();
        return refuse(call + ": the detector is on another device than the media guard");
    }
    mww_detector_layout layout;
    mww_get_detector_layout(det, &layout);
    if (model >= layout.n_models)
        return refuse(call + ": model " + std::to_string(model) + " of a detector of " + std::to_string(layout.n_models) + " model(s)");
    DeviceGuard guard(g->device);
    if (guard.err != cudaSuccess) return cuda_fail(nullptr, guard.err, "cudaSetDevice");
    MediaSlotsArgs sa{};
    sa.n = capacity; sa.n_streams = info.n_streams; sa.C = C; sa.n_samples = g->rule.n_samples; sa.seen = S;
    sa.count = d_count; sa.events = d_events; sa.positions = reinterpret_cast<const long long *>(d_positions);
    sa.ev_group = detector_event_groups(det);
    sa.capacity = capacity; sa.model = model < 0 ? -1 : model; sa.post = post;
    return run(g, src, sa, d_confirmed, d_matches, d_media, d_passed, st, call);
}

int mww_media_register(mww_media_guard_t *g, const int16_t *d_audio, int n_samples, int *index, void *cu_stream) {
    const std::string call = "mww_media_register: ";
    if (!g || !d_audio) return refuse(call + "needs a media guard and audio");
    const int k = g->n_clips;
    if (k >= g->rule.max_media) return refuse(call + "the guard holds " + std::to_string(g->rule.max_media) + " registered clips already (max_media)");
    if (n_samples < kMediaMinSamples || n_samples > g->rule.max_media_samples)
        return refuse(call + "n_samples must be in [640, " + std::to_string(g->rule.max_media_samples) + "] (max_media_samples)");
    const int T = frames_of(n_samples), W = T - 1;
    if (W < g->rule.min_overlap) return refuse(call + "the clip gives " + std::to_string(W) + " fingerprint words, fewer than min_overlap");
    DeviceGuard guard(g->device);
    if (guard.err != cudaSuccess) return cuda_fail(nullptr, guard.err, "cudaSetDevice");
    cudaStream_t st = static_cast<cudaStream_t>(cu_stream);
    if (int rc = mww_reset(g->hm, nullptr, 0, st)) return pass_on(rc, g->hm, call + "frontend reset");
    int rows = 0;
    if (int rc = mww_features(g->hm, d_audio, n_samples, n_samples, g->m_feat, g->clip_frames, &rows, st)) return pass_on(rc, g->hm, call + "features");
    GCU(launch_media_fingerprint(g->m_feat, g->clip_frames, 1, W, g->clip_fp + g->clip_words, W, st));
    g->launches += 1;
    // entry k of the host copies is past n_clips, so nothing reads it until the guard counts the clip, after the copies
    const long long tasks = g->clip_tasks + media_clip_tasks(g->words, W, g->rule.min_overlap);
    g->h_off[k] = g->clip_words;
    g->h_len[k] = W;
    g->h_task0[k] = (int32_t)g->clip_tasks;
    g->h_task0[k + 1] = (int32_t)tasks;
    GCU(cudaMemcpyAsync(g->clip_off + k, &g->h_off[k], sizeof(long long), cudaMemcpyHostToDevice, st));
    GCU(cudaMemcpyAsync(g->clip_len + k, &g->h_len[k], sizeof(int32_t), cudaMemcpyHostToDevice, st));
    GCU(cudaMemcpyAsync(g->clip_task0 + k, &g->h_task0[k], 2 * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    g->clip_words += W;
    g->clip_tasks = tasks;
    g->n_clips = k + 1;
    if (index) *index = k;
    return MWW_OK;
}

int mww_media_clear_registered(mww_media_guard_t *g) {
    if (!g) return refuse("mww_media_clear_registered: media guard is NULL");
    std::fill(g->h_len.begin(), g->h_len.end(), 0);
    std::fill(g->h_off.begin(), g->h_off.end(), 0);
    std::fill(g->h_task0.begin(), g->h_task0.end(), 0);
    g->clip_words = g->clip_tasks = 0;
    g->n_clips = 0;
    return MWW_OK;
}

int mww_media_clear_ring(mww_media_guard_t *g) {
    if (!g) return refuse("mww_media_clear_ring: media guard is NULL");
    DeviceGuard guard(g->device);
    if (guard.err != cudaSuccess) return cuda_fail(nullptr, guard.err, "cudaSetDevice");
    GCU(cudaDeviceSynchronize());
    GCU(cudaMemset(g->state, 0, sizeof(MediaRingState)));
    GCU(cudaDeviceSynchronize());
    return MWW_OK;
}

int mww_media_get_state(mww_media_guard_t *g, void *h_state, long long *n_bytes) {
    const std::string call = "mww_media_get_state: ";
    if (!g || !n_bytes) return refuse(call + "needs a media guard and n_bytes");
    const int n_media = g->n_clips;
    const long long need = state_bytes(g, n_media, g->clip_words);
    if (!h_state) { *n_bytes = need; return MWW_OK; }
    if (*n_bytes < need) return refuse(call + "the buffer holds " + std::to_string(*n_bytes) + " bytes; the state is " + std::to_string(need));
    DeviceGuard guard(g->device);
    if (guard.err != cudaSuccess) return cuda_fail(nullptr, guard.err, "cudaSetDevice");
    GCU(cudaDeviceSynchronize());
    MediaRingState s{};
    GCU(cudaMemcpy(&s, g->state, sizeof(s), cudaMemcpyDeviceToHost));
    char *p = static_cast<char *>(h_state);
    const long long R = g->rule.ring, W = g->words;
    const int32_t hdr[4] = {g->words, g->rule.ring, n_media, 0};
    std::memcpy(p, &s.count, 8);
    std::memcpy(p + 8, hdr, 16);
    std::memcpy(p + 24, &g->clip_words, 8);
    p += 32;
    if (R > 0) {
        GCU(cudaMemcpy(p, g->ring_fp, R * W * 8, cudaMemcpyDeviceToHost)); p += R * W * 8;
        GCU(cudaMemcpy(p, g->ring_pos, R * 8, cudaMemcpyDeviceToHost)); p += R * 8;
        GCU(cudaMemcpy(p, g->ring_stream, R * 4, cudaMemcpyDeviceToHost)); p += R * 4;
        GCU(cudaMemcpy(p, g->ring_hh, R * 4, cudaMemcpyDeviceToHost)); p += R * 4;
    }
    for (int k = 0; k < n_media; ++k) { const long long w = g->h_len[k]; std::memcpy(p, &w, 8); p += 8; }
    if (g->clip_words > 0) GCU(cudaMemcpy(p, g->clip_fp, g->clip_words * 8, cudaMemcpyDeviceToHost));
    *n_bytes = need;
    return MWW_OK;
}

int mww_media_set_state(mww_media_guard_t *g, const void *h_state, long long n_bytes) {
    const std::string call = "mww_media_set_state: ";
    if (!g || !h_state) return refuse(call + "needs a media guard and a state");
    if (n_bytes < 32) return refuse(call + "the state is shorter than its header");
    const char *p = static_cast<const char *>(h_state);
    long long count = 0, media_words = 0;
    int32_t hdr[4];
    std::memcpy(&count, p, 8);
    std::memcpy(hdr, p + 8, 16);
    std::memcpy(&media_words, p + 24, 8);
    if (hdr[0] != g->words || hdr[1] != g->rule.ring)
        return refuse(call + "the state is of a guard with other fingerprint words or another ring size");
    const int n_media = hdr[2];
    if (count < 0) return refuse(call + "ring_count must not be negative");
    if (n_media < 0 || n_media > g->rule.max_media) return refuse(call + "more registered clips than max_media");
    if (media_words < 0 || media_words > (long long)g->rule.max_media * std::max(g->clip_frames - 1, 0))
        return refuse(call + "media_words out of range");
    if (n_bytes != state_bytes(g, n_media, media_words)) return refuse(call + "the state's size does not match its header");
    const long long R = g->rule.ring, W = g->words;
    const char *lens = p + 32 + R * W * 8 + R * 16;
    std::vector<long long> len(n_media);
    long long sum = 0;
    for (int k = 0; k < n_media; ++k) {
        std::memcpy(&len[k], lens + 8 * k, 8);
        if (len[k] < g->rule.min_overlap || len[k] > g->clip_frames - 1) return refuse(call + "a registered clip's length is out of range");
        sum += len[k];
    }
    if (sum != media_words) return refuse(call + "the registered clips' lengths do not add up to media_words");
    DeviceGuard guard(g->device);
    if (guard.err != cudaSuccess) return cuda_fail(nullptr, guard.err, "cudaSetDevice");
    GCU(cudaDeviceSynchronize());
    const MediaRingState s{count, 0, 0};
    GCU(cudaMemcpy(g->state, &s, sizeof(s), cudaMemcpyHostToDevice));
    p += 32;
    if (R > 0) {
        GCU(cudaMemcpy(g->ring_fp, p, R * W * 8, cudaMemcpyHostToDevice)); p += R * W * 8;
        GCU(cudaMemcpy(g->ring_pos, p, R * 8, cudaMemcpyHostToDevice)); p += R * 8;
        GCU(cudaMemcpy(g->ring_stream, p, R * 4, cudaMemcpyHostToDevice)); p += R * 4;
        GCU(cudaMemcpy(g->ring_hh, p, R * 4, cudaMemcpyHostToDevice)); p += R * 4;
    }
    p += 8LL * n_media;
    mww_media_clear_registered(g);
    for (int k = 0; k < n_media; ++k) {
        g->h_off[k] = g->clip_words;
        g->h_len[k] = (int32_t)len[k];
        g->h_task0[k] = (int32_t)g->clip_tasks;
        g->clip_words += len[k];
        g->clip_tasks += media_clip_tasks(g->words, (int)len[k], g->rule.min_overlap);
        g->h_task0[k + 1] = (int32_t)g->clip_tasks;
    }
    g->n_clips = n_media;
    if (media_words > 0) GCU(cudaMemcpy(g->clip_fp, p, media_words * 8, cudaMemcpyHostToDevice));
    const size_t M = (size_t)g->rule.max_media;
    if (M > 0) {
        GCU(cudaMemcpy(g->clip_off, g->h_off.data(), M * sizeof(long long), cudaMemcpyHostToDevice));
        GCU(cudaMemcpy(g->clip_len, g->h_len.data(), M * sizeof(int32_t), cudaMemcpyHostToDevice));
    }
    GCU(cudaMemcpy(g->clip_task0, g->h_task0.data(), (M + 1) * sizeof(int32_t), cudaMemcpyHostToDevice));
    return MWW_OK;
}

}  // extern "C"
