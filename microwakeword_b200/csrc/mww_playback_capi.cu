// mww_playback_capi.cu -- the extern "C" entry points of the playback guard (include/mww.h, "playback guard").  Host code only:
// the kernels are in mww_playback.{h,cu}.  A guard is bound to a handle whose history axis it uses; it reads that handle's
// counters on the host (history_ring) and never launches work on it.  It scores reference clips on a verifier of its own
// through the verifier's scoring pass (verifier_score_clips), and its messages go to mww_last_error(NULL).
//
// The row map and the heads are mirrored on the host, because a write's ids and starts come from the host: a write plans its
// jobs from the mirror, stages them in one copy, and updates the mirror only once the copy and the launch are enqueued.
#include <algorithm>
#include <string>
#include <vector>

#include "mww_capi.h"
#include "mww_kernels.h"

using namespace mww;

struct mww_playback_guard {
    const mww_t *h = nullptr;           // the bound handle
    int device = 0, slots = 0, rows = 0, C = 0, n_streams = 0, L = 0;
    mww_playback_rule rule{};
    long long launches = 0;             // the guard's own kernel launches
    mww_verifier_t *v = nullptr;        // the model on `slots` streams with n_samples = L_ref: its clip buffer takes the reference clips
    int16_t *ring = nullptr;            // [rows][C]
    int32_t *row_of = nullptr;          // [n_streams] stream -> row, -1: none
    long long *head = nullptr;          // [rows]
    PlaybackJob *d_jobs = nullptr;      // [n_streams + rows]
    int32_t *sid = nullptr, *heard = nullptr;   // [slots]
    std::vector<int32_t> h_row_of, h_stream_of;   // host mirror: [n_streams], [rows] (-1: free)
    std::vector<long long> h_head;                // [rows]
    std::vector<PlaybackJob> jobs;                // [n_streams + rows] staging of one call's jobs
    std::vector<char> listed;                     // [n_streams] the ids of the current call
};

namespace {

#define PCU(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return cuda_fail(nullptr, e_, #call); } while (0)

int refuse(const std::string &msg) { return fail(nullptr, MWW_EINVAL, msg); }

void guard_free(mww_playback_guard_t *g) {
    if (g->v) mww_verifier_destroy(g->v);
    cudaFree(g->ring); cudaFree(g->row_of); cudaFree(g->head); cudaFree(g->d_jobs); cudaFree(g->sid); cudaFree(g->heard);
    delete g;
}

int guard_alloc(mww_playback_guard_t *g) {
    const size_t R = (size_t)g->rows, N = (size_t)g->n_streams, S = (size_t)g->slots;
    PCU(cudaMalloc(&g->ring, R * g->C * sizeof(int16_t)));
    PCU(cudaMalloc(&g->row_of, N * sizeof(int32_t)));
    PCU(cudaMalloc(&g->head, R * sizeof(long long)));
    PCU(cudaMalloc(&g->d_jobs, (N + R) * sizeof(PlaybackJob)));
    PCU(cudaMalloc(&g->sid, S * sizeof(int32_t)));
    PCU(cudaMalloc(&g->heard, S * sizeof(int32_t)));
    PCU(cudaMemset(g->row_of, 0xff, N * sizeof(int32_t)));
    PCU(cudaMemset(g->head, 0, R * sizeof(long long)));
    PCU(cudaDeviceSynchronize());
    g->h_row_of.assign(N, -1);
    g->h_stream_of.assign(R, -1);
    g->h_head.assign(R, 0);
    g->jobs.assign(N + R, PlaybackJob{});
    g->listed.assign(N, 0);
    return MWW_OK;
}

// the bound handle's history as the guard reads it: refused when it keeps none or is poisoned
int bound_history(const mww_playback_guard_t *g, const std::string &call, HistoryRing *hr) {
    *hr = history_ring(g->h);
    if (!hr->ring) return refuse(call + ": the bound handle keeps no audio history");
    if (hr->poisoned) return refuse(call + ": the bound handle cannot be read: a staged call failed on it");
    return MWW_OK;
}

// The checks both check calls share, before any device work
int check_guard(const mww_playback_guard_t *g, const std::string &call, int n, HistoryRing *hr) {
    if (!g) return refuse(call + ": needs a playback guard");
    if (n < 0 || n > g->slots) return refuse(call + ": " + std::to_string(n) + " slots for a playback guard of " + std::to_string(g->slots));
    return bound_history(g, call, hr);
}

// The pass over n slots: the slots kernel with the reference read into the verifier's clip buffer, the verifier's scoring pass
// and the decision.  A constant number of launches for n >= 1.
int run(mww_playback_guard_t *g, PlaybackSlotsArgs a, const int32_t *d_confirmed, float *d_scores, int32_t *d_flagged, int32_t *d_passed,
        cudaStream_t st, const std::string &call) {
    a.n_streams = g->n_streams; a.C = g->C; a.L = g->L; a.min_delay = g->rule.min_delay;
    a.ring = g->ring; a.row_of = g->row_of; a.head = g->head;
    a.out = verifier_clips(g->v); a.out_stride = g->L;
    a.sid = g->sid; a.heard = g->heard;
    PCU(launch_playback_slots(a, st));
    if (int rc = verifier_score_clips(g->v, a.n, st, call)) return rc;
    PCU(launch_playback_decide(a.n, g->sid, g->heard, verifier_scores(g->v), g->rule.cutoff, d_confirmed, d_scores, d_flagged, d_passed, st));
    g->launches += 2;
    return MWW_OK;
}

}  // namespace

extern "C" {

int mww_playback_guard_create(const mww_t *h, const void *model_blob, size_t n_bytes, int slots, int rows, int capacity,
                              const mww_playback_rule *rule, mww_playback_guard_t **out) {
    const std::string call = "mww_playback_guard_create: ";
    if (!out) return refuse(call + "out is NULL");
    *out = nullptr;
    if (!rule) return refuse(call + "rule is NULL");
    const mww_playback_rule &r = *rule;
    if (slots < 1) return refuse(call + "slots must be at least 1");
    if (capacity < 8 || capacity > kPlaybackMaxSamples || capacity % 8 != 0) return refuse(call + "capacity must be a multiple of 8 in [8, 2^22]");
    if (r.n_samples < kWindow) return refuse(call + "n_samples must be at least 480");
    if (r.min_delay < 0 || r.min_delay > r.max_delay || r.max_delay > kPlaybackMaxSamples)
        return refuse(call + "the delays must satisfy 0 <= min_delay <= max_delay <= 2^22");
    const long long L = (long long)r.n_samples + r.max_delay - r.min_delay;
    if (L > std::min(capacity, kPlaybackMaxSamples))
        return refuse(call + "L_ref = n_samples + max_delay - min_delay = " + std::to_string(L) + " must be at most min(capacity, 2^22)");
    if (!model_blob || n_bytes == 0) return refuse(call + "a playback guard needs a model (the blob is NULL)");
    if (!h) return refuse(call + "needs a handle");
    int cap = 0;
    mww_get_audio_history(h, &cap, nullptr);
    if (cap == 0) return refuse(call + "the handle keeps no audio history (mww_set_audio_history): the guard uses its axis");
    if (mww_model_count(h) == 0) return refuse(call + "the handle is frontend-only");
    mww_info info;
    if (mww_get_info(h, &info) != MWW_OK) return refuse(call + "cannot read the handle");
    if (rows < 1 || rows > info.n_streams) return refuse(call + "rows must be in [1, " + std::to_string(info.n_streams) + "] (the handle's streams)");
    mww_playback_guard_t *g = new mww_playback_guard;
    g->h = h; g->device = info.device; g->slots = slots; g->rows = rows; g->C = capacity; g->n_streams = info.n_streams; g->L = (int)L;
    g->rule = r; g->rule.pad = 0;
    // the verifier's own refusals (window, ignore_steps, cutoff, every score NaN) and its model, on the handle's device
    const mww_verify_rule vr{(int32_t)L, r.window, r.ignore_steps, 0, r.cutoff};
    if (int rc = mww_verifier_create(model_blob, n_bytes, info.device, slots, &vr, &g->v)) { guard_free(g); return rc; }
    DeviceGuard guard(info.device);
    if (guard.err != cudaSuccess) { guard_free(g); return cuda_fail(nullptr, guard.err, "cudaSetDevice"); }
    if (int rc = guard_alloc(g)) { guard_free(g); return rc; }
    *out = g;
    return MWW_OK;
}

int mww_playback_guard_destroy(mww_playback_guard_t *g) {
    if (!g) return MWW_OK;
    DeviceGuard guard(g->device);
    cudaDeviceSynchronize();
    guard_free(g);
    return MWW_OK;
}

int mww_playback_guard_info(const mww_playback_guard_t *g, mww_playback_guard_desc *out) {
    if (!g || !out) return refuse("mww_playback_guard_info: needs a playback guard and out");
    mww_verifier_desc vd;
    mww_verifier_info(g->v, &vd);
    *out = mww_playback_guard_desc{};
    out->slots = g->slots; out->steps = vd.steps; out->rows = g->rows;
    out->rows_used = (int32_t)std::count_if(g->h_stream_of.begin(), g->h_stream_of.end(), [](int32_t s) { return s >= 0; });
    out->capacity = g->C; out->l_ref = g->L; out->device = g->device; out->rule = g->rule;
    out->launches = g->launches + vd.launches;
    return MWW_OK;
}

int mww_playback_write(mww_playback_guard_t *g, const int32_t *h_ids, const long long *h_starts, int n, const int16_t *d_audio, int n_samples,
                       long long audio_stride, void *cu_stream) {
    const std::string call = "mww_playback_write";
    if (!g) return refuse(call + ": needs a playback guard");
    if (n < 0) return refuse(call + ": n must not be negative");
    if (n_samples < 0 || n_samples > kPlaybackMaxSamples) return refuse(call + ": n_samples must be in [0, 2^22]");
    if (audio_stride < n_samples) return refuse(call + ": audio_stride must be at least n_samples");
    if (n > 0 && (!h_ids || !h_starts)) return refuse(call + ": h_ids and h_starts must not be NULL");
    if (n > 0 && n_samples > 0 && !d_audio) return refuse(call + ": d_audio is NULL");
    HistoryRing hr;
    if (int rc = bound_history(g, call, &hr)) return rc;
    int bad = -1;
    for (int i = 0; i < n && bad < 0; ++i) {
        if (h_ids[i] < 0 || h_ids[i] >= g->n_streams) bad = 0;
        else if (g->listed[h_ids[i]]) bad = 1;
        else if (h_starts[i] < -kPlaybackMaxStart || h_starts[i] > kPlaybackMaxStart) bad = 2;
        else g->listed[h_ids[i]] = 1;
    }
    auto unlist = [&] { for (int i = 0; i < n; ++i) if (h_ids[i] >= 0 && h_ids[i] < g->n_streams) g->listed[h_ids[i]] = 0; };
    if (bad >= 0) {
        unlist();
        static const char *why[] = {"an id is outside [0, n_streams)", "an id is listed twice", "a start is outside [-2^50, 2^50]"};
        return refuse(call + ": " + why[bad]);
    }
    const long long S = hr.seen;
    const int n_jobs = playback_plan(h_ids, h_starts, n, S, g->C, g->rows, g->h_row_of.data(), g->h_stream_of.data(), g->h_head.data(),
                                     g->listed.data(), g->jobs.data());
    unlist();
    if (n_jobs < 0) return fail(nullptr, MWW_ENOMEM, call + ": the write needs more rows than are free (rows = " + std::to_string(g->rows) + ")");
    if (n_jobs == 0) return MWW_OK;
    DeviceGuard guard(g->device);
    if (guard.err != cudaSuccess) return cuda_fail(nullptr, guard.err, "cudaSetDevice");
    cudaStream_t st = static_cast<cudaStream_t>(cu_stream);
    PCU(cudaMemcpyAsync(g->d_jobs, g->jobs.data(), (size_t)n_jobs * sizeof(PlaybackJob), cudaMemcpyHostToDevice, st));
    PCU(launch_playback_write(g->d_jobs, n_jobs, d_audio, audio_stride, n_samples, g->ring, g->C, g->row_of, g->head, st));
    g->launches += 1;
    playback_commit(g->jobs.data(), n, n_samples, S, g->C, g->rows, g->h_row_of.data(), g->h_stream_of.data(), g->h_head.data());
    return MWW_OK;
}

int mww_playback_read(mww_playback_guard_t *g, const int32_t *d_ids, const long long *d_ends, int n, int n_samples, int16_t *d_out,
                      long long out_stride, void *cu_stream) {
    const std::string call = "mww_playback_read";
    if (!g) return refuse(call + ": needs a playback guard");
    if (n < 0) return refuse(call + ": n must not be negative");
    if (n_samples < 0 || n_samples > kPlaybackMaxSamples) return refuse(call + ": n_samples must be in [0, 2^22]");
    if (out_stride < n_samples) return refuse(call + ": out_stride must be at least n_samples");
    if (n > 0 && n_samples > 0 && (!d_ids || !d_ends || !d_out)) return refuse(call + ": d_ids, d_ends and d_out must not be NULL");
    if (n == 0 || n_samples == 0) return MWW_OK;
    DeviceGuard guard(g->device);
    if (guard.err != cudaSuccess) return cuda_fail(nullptr, guard.err, "cudaSetDevice");
    PlaybackSlotsArgs a{};
    a.n = n; a.n_streams = g->n_streams; a.C = g->C; a.L = n_samples;
    a.ids = d_ids; a.ends = d_ends;
    a.ring = g->ring; a.row_of = g->row_of; a.head = g->head;
    a.out = d_out; a.out_stride = out_stride;
    PCU(launch_playback_slots(a, static_cast<cudaStream_t>(cu_stream)));
    g->launches += 1;
    return MWW_OK;
}

int mww_playback_reset(mww_playback_guard_t *g, const int32_t *h_ids, int n, void *cu_stream) {
    const std::string call = "mww_playback_reset";
    if (!g) return refuse(call + ": needs a playback guard");
    if (h_ids && n < 0) return refuse(call + ": n must not be negative");
    if (h_ids)
        for (int i = 0; i < n; ++i)
            if (h_ids[i] < 0 || h_ids[i] >= g->n_streams) return refuse(call + ": an id is outside [0, n_streams)");
    DeviceGuard guard(g->device);
    if (guard.err != cudaSuccess) return cuda_fail(nullptr, guard.err, "cudaSetDevice");
    cudaStream_t st = static_cast<cudaStream_t>(cu_stream);
    if (!h_ids) {
        PCU(cudaMemsetAsync(g->row_of, 0xff, (size_t)g->n_streams * sizeof(int32_t), st));
        std::fill(g->h_row_of.begin(), g->h_row_of.end(), -1);
        std::fill(g->h_stream_of.begin(), g->h_stream_of.end(), -1);
        return MWW_OK;
    }
    int n_jobs = 0;
    for (int i = 0; i < n; ++i)
        if (g->h_row_of[h_ids[i]] >= 0 && !g->listed[h_ids[i]]) { g->listed[h_ids[i]] = 1; g->jobs[n_jobs++] = PlaybackJob{h_ids[i], -1, 0, 0}; }
    for (int j = 0; j < n_jobs; ++j) g->listed[g->jobs[j].stream] = 0;
    if (n_jobs == 0) return MWW_OK;
    PCU(cudaMemcpyAsync(g->d_jobs, g->jobs.data(), (size_t)n_jobs * sizeof(PlaybackJob), cudaMemcpyHostToDevice, st));
    PCU(launch_playback_write(g->d_jobs, n_jobs, nullptr, 0, 0, g->ring, g->C, g->row_of, g->head, st));
    g->launches += 1;
    for (int j = 0; j < n_jobs; ++j) {
        const int32_t s = g->jobs[j].stream;
        g->h_stream_of[g->h_row_of[s]] = -1;
        g->h_row_of[s] = -1;
    }
    return MWW_OK;
}

int mww_playback_get_heads(const mww_playback_guard_t *g, int32_t *h_rows, int64_t *h_heads) {
    if (!g) return refuse("mww_playback_get_heads: needs a playback guard");
    for (int s = 0; s < g->n_streams; ++s) {
        const int32_t r = g->h_row_of[s];
        if (h_rows) h_rows[s] = r;
        if (h_heads) h_heads[s] = r >= 0 ? g->h_head[r] : 0;
    }
    return MWW_OK;
}

int mww_playback_check_streams(mww_playback_guard_t *g, const int32_t *d_ids, const long long *d_ends, int n, const int32_t *d_confirmed,
                               float *d_scores, int32_t *d_flagged, int32_t *d_passed, void *cu_stream) {
    const std::string call = "mww_playback_check_streams";
    HistoryRing hr;
    if (int rc = check_guard(g, call, n, &hr)) return rc;
    if (n > 0 && (!d_ids || !d_ends)) return refuse(call + ": d_ids and d_ends must not be NULL");
    if (n == 0) return MWW_OK;
    DeviceGuard guard(g->device);
    if (guard.err != cudaSuccess) return cuda_fail(nullptr, guard.err, "cudaSetDevice");
    PlaybackSlotsArgs a{};
    a.n = n; a.seen = hr.seen; a.ids = d_ids; a.ends = d_ends;
    return run(g, a, d_confirmed, d_scores, d_flagged, d_passed, static_cast<cudaStream_t>(cu_stream), call);
}

int mww_playback_check_detections_at(mww_playback_guard_t *g, mww_detector_t *det, int model, long long post, const int32_t *d_confirmed,
                                     float *d_scores, int32_t *d_flagged, int32_t *d_passed, void *cu_stream) {
    const std::string call = "mww_playback_check_detections_at";
    if (!g) return refuse(call + ": needs a playback guard");
    if (!det) return refuse(call + ": detector is NULL");
    if (post < 0 || post > kPlaybackMaxSamples) return refuse(call + ": post must be in [0, 2^22]");
    const int64_t *d_positions = nullptr;
    if (mww_get_detector_positions(det, &d_positions) != MWW_OK)
        return refuse(call + ": the detector is not timed (mww_time_detector_events): its events carry no positions");
    const long long *d_count = nullptr;
    const mww_event *d_events = nullptr;
    int capacity = 0;
    mww_detector_buffers(det, &d_count, &d_events, nullptr, &capacity);
    if (capacity > g->slots)
        return refuse(call + ": the detector keeps " + std::to_string(capacity) + " events; the playback guard has " + std::to_string(g->slots) + " slots");
    HistoryRing hr;
    if (int rc = check_guard(g, call, capacity, &hr)) return rc;
    cudaPointerAttributes attr;
    if (cudaPointerGetAttributes(&attr, d_count) != cudaSuccess || attr.device != g->device) {
        cudaGetLastError();
        return refuse(call + ": the detector is on another device than the playback guard");
    }
    mww_detector_layout layout;
    mww_get_detector_layout(det, &layout);
    if (model >= layout.n_models)
        return refuse(call + ": model " + std::to_string(model) + " of a detector of " + std::to_string(layout.n_models) + " model(s)");
    DeviceGuard guard(g->device);
    if (guard.err != cudaSuccess) return cuda_fail(nullptr, guard.err, "cudaSetDevice");
    PlaybackSlotsArgs a{};
    a.n = capacity; a.seen = hr.seen;
    a.count = d_count; a.events = d_events; a.positions = reinterpret_cast<const long long *>(d_positions);
    a.capacity = capacity; a.model = model < 0 ? -1 : model; a.post = post;
    return run(g, a, d_confirmed, d_scores, d_flagged, d_passed, static_cast<cudaStream_t>(cu_stream), call);
}

}  // extern "C"
