// mww_endpoint_capi.cu -- the extern "C" entry points of the endpointer (include/mww.h, "endpointing").  Host code only: the
// four kernels are in mww_endpoint.{h,cu}.  An endpointer is an object of its own, like a detector: it reads its handle's
// counters through public calls and its history ring through history_ring (mww_capi.h), launches nothing on the handle, and
// its messages go to mww_last_error(NULL).
#include <algorithm>
#include <cmath>
#include <string>
#include <vector>

#include "mww_capi.h"
#include "mww_kernels.h"

using namespace mww;

struct mww_endpointer {
    int device = 0, model = 0, stride = 1, hop = kHop, n_streams = 0, capacity = 0;
    const mww_t *h = nullptr;
    EndpointArgs a{};                     // the rule and every device pointer, as the kernels take them
    std::vector<int32_t> members;         // row -> global id
    std::vector<int32_t> row_of;          // global id -> row, -1 for a non-member
    int32_t *d_ids = nullptr;             // [n_rows] a host id list, filtered to members without repeats
    int32_t *d_rec_ids = nullptr;         // [rec_ids_cap] the id list of a record call, as given
    size_t rec_ids_cap = 0;
    long long launches = 0;
    int tag = 0;                          // arm calls so far
    // the handle's counters after the last update or whole reset, the steps consumed since then and their last positions
    long long base_seen = 0, steps = 0;
    int base_buffered = 0, base_pending = 0;
    long long pos[kEndpointMaxLookback] = {};   // pos[i]: the step i steps before the newest
    // the positioned forms (include/mww.h, "positioned arm"): each row's mute word, the reduction keys of arm_at and the
    // staging buffer of a host position list, all [n_rows]; positioned switches on for good at the first arm_at, set_mutes or
    // import of positioned records, and selects the kernels of libmww_endpoint_at.so from then on
    int32_t *d_mute = nullptr;
    unsigned long long *d_at_key = nullptr;
    long long *d_positions = nullptr;
    bool positioned = false;
};

namespace {

#define ECU(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return cuda_fail(nullptr, e_, #call); } while (0)

int refuse(const std::string &msg) { return fail(nullptr, MWW_EINVAL, msg); }

void endpointer_free(mww_endpointer_t *ep) {
    EndpointArgs &a = ep->a;
    cudaFree(a.hist); cudaFree(a.seen); cudaFree(a.flags); cudaFree(a.armed); cudaFree(a.elapsed); cudaFree(a.run); cudaFree(a.silence);
    cudaFree(a.heard); cudaFree(a.start); cudaFree(a.speech_end); cudaFree(a.arm_tag); cudaFree((void *)a.row_of); cudaFree(a.count);
    cudaFree(a.events); cudaFree(a.ended); cudaFree(ep->d_ids); cudaFree(ep->d_rec_ids);
    cudaFree(ep->d_mute); cudaFree(ep->d_at_key); cudaFree(ep->d_positions);
    delete ep;
}

template <typename T>
cudaError_t alloc_fill(T **p, size_t n, int byte) {
    cudaError_t e = cudaMalloc(p, std::max<size_t>(n, 1) * sizeof(T));
    return e == cudaSuccess ? cudaMemset(*p, byte, std::max<size_t>(n, 1) * sizeof(T)) : e;
}

int endpointer_alloc(mww_endpointer_t *ep) {
    EndpointArgs &a = ep->a;
    const size_t R = (size_t)a.n_rows, W = (size_t)(a.rule.vad_window - 1);
    ECU(alloc_fill(&a.hist, W * R, 0));
    ECU(alloc_fill(&a.seen, R, 0));
    ECU(alloc_fill(&a.flags, R, 0));
    ECU(alloc_fill(&a.armed, R, 0xFF));
    ECU(alloc_fill(&a.elapsed, R, 0));
    ECU(alloc_fill(&a.run, R, 0));
    ECU(alloc_fill(&a.silence, R, 0));
    ECU(alloc_fill(&a.heard, R, 0));
    ECU(alloc_fill(&a.start, R, 0));
    ECU(alloc_fill(&a.speech_end, R, 0));
    ECU(alloc_fill(&a.arm_tag, R, 0));
    int32_t *row_of = nullptr;
    ECU(alloc_fill(&row_of, (size_t)ep->n_streams, 0));
    a.row_of = row_of;
    ECU(cudaMemcpy(row_of, ep->row_of.data(), ep->row_of.size() * sizeof(int32_t), cudaMemcpyHostToDevice));
    ECU(alloc_fill(&a.count, 1, 0));
    ECU(alloc_fill(&a.events, (size_t)a.capacity, 0));
    ECU(alloc_fill(&a.ended, (size_t)a.capacity, 0xFF));
    ECU(alloc_fill(&ep->d_ids, R, 0));
    ECU(alloc_fill(&ep->d_mute, R, 0));
    ECU(alloc_fill(&ep->d_at_key, R, 0));
    ECU(alloc_fill(&ep->d_positions, R, 0));
    ECU(cudaDeviceSynchronize());
    return MWW_OK;
}

// the handle's counters the time axis is read from: samples_seen, frontend_buffered and model k's pending rows
int read_counters(const mww_endpointer_t *ep, long long *seen, int *buffered, int *pending) {
    mww_info info, mi;
    int cap = 0;
    if (mww_get_info(ep->h, &info) != MWW_OK || mww_get_model_info(ep->h, ep->model, &mi) != MWW_OK ||
        mww_get_audio_history(ep->h, &cap, seen) != MWW_OK)
        return refuse("the endpointer's handle cannot be read");
    *buffered = info.frontend_buffered;
    *pending = mi.pending_rows;
    return MWW_OK;
}

// the host list of a call, filtered to members of the set without repeats (so it fits the [n_rows] staging buffer), on the device
int stage_ids(mww_endpointer_t *ep, const std::string &call, const int32_t *h_ids, int n, int *n_out, cudaStream_t st) {
    if (n < 0 || (n > 0 && !h_ids)) return refuse(call + ": needs n >= 0 and ids with n > 0");
    std::vector<int32_t> ids;
    std::vector<char> listed(ep->members.size(), 0);
    for (int i = 0; i < n; ++i) {
        if (h_ids[i] < 0 || h_ids[i] >= ep->n_streams)
            return refuse(call + ": stream id " + std::to_string(h_ids[i]) + " out of range [0, " + std::to_string(ep->n_streams) + ")");
        const int r = ep->row_of[h_ids[i]];
        if (r >= 0 && !listed[r]) { listed[r] = 1; ids.push_back(h_ids[i]); }
    }
    // from pageable memory, as mww_reset's list: the copy has taken the bytes when cudaMemcpyAsync returns
    if (!ids.empty()) ECU(cudaMemcpyAsync(ep->d_ids, ids.data(), ids.size() * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    *n_out = (int)ids.size();
    return MWW_OK;
}

EndpointReplay replay_of(mww_endpointer_t *ep) {
    EndpointReplay R{};
    R.steps = (int)std::min<long long>(ep->a.rule.lookback_steps, ep->steps);
    R.tag = ++ep->tag;
    for (int i = 0; i < kEndpointMaxLookback; ++i) R.pos[i] = ep->pos[i];
    return R;
}

int arm(mww_endpointer_t *ep, const int32_t *d_ids, int n, cudaStream_t st) {
    DeviceGuard guard(ep->device);
    if (guard.err != cudaSuccess) return cuda_fail(nullptr, guard.err, "cudaSetDevice");
    if (ep->positioned) ECU(launch_endpoint_arm_muted(ep->a, replay_of(ep), ep->d_mute, d_ids, n, st));
    else ECU(launch_endpoint_arm(ep->a, replay_of(ep), d_ids, n, st));
    ep->launches += 1;
    return MWW_OK;
}

// the position of the newest step consumed (or of where it would have been, with none since a whole reset)
long long newest_position(const mww_endpointer_t *ep) {
    return endpoint_position(ep->base_seen, ep->base_buffered, ep->hop, ep->base_pending, ep->stride, 1, 0);
}

// arm_at: two launches, the reduction of each row's latest position and the arm; the endpointer is positioned from here on
int arm_at(mww_endpointer_t *ep, const int32_t *d_ids, const long long *d_positions, int n, long long skip, cudaStream_t st) {
    DeviceGuard guard(ep->device);
    if (guard.err != cudaSuccess) return cuda_fail(nullptr, guard.err, "cudaSetDevice");
    ep->positioned = true;
    EndpointAt A{};
    A.R = replay_of(ep);
    A.q = newest_position(ep);
    A.skip = skip;
    A.mute = ep->d_mute;
    A.key = ep->d_at_key;
    ECU(launch_endpoint_arm_at(ep->a, A, d_ids, d_positions, n, st));
    ep->launches += 2;
    return MWW_OK;
}

int check_skip(const std::string &call, long long skip) {
    if (skip < 0 || skip > kHistoryMaxCapacity) return refuse(call + ": skip_samples must be in [0, 2^22]");
    return MWW_OK;
}

int clear(mww_endpointer_t *ep, const int32_t *d_ids, int n, int reset, cudaStream_t st) {
    DeviceGuard guard(ep->device);
    if (guard.err != cudaSuccess) return cuda_fail(nullptr, guard.err, "cudaSetDevice");
    if (ep->positioned) ECU(launch_endpoint_clear_muted(ep->a, ep->d_mute, d_ids, n, reset, st));
    else ECU(launch_endpoint_clear(ep->a, d_ids, n, reset, st));
    ep->launches += 1;
    return MWW_OK;
}

// ---- endpointer records (layout and per-row bodies: mww_serving_records.h) ----
void fill_layout(const mww_endpointer_t *ep, mww_endpointer_layout *out) {
    *out = mww_endpointer_layout{};
    out->record_bytes = endpoint_record_layout(ep->a.rule.vad_window).record_bytes;
    out->vad_window = ep->a.rule.vad_window; out->stride = ep->stride; out->hop_samples = ep->hop;
    out->buffered = ep->base_buffered; out->pending = ep->base_pending;
    out->samples_seen = ep->base_seen; out->steps = ep->steps;
    out->pad = ep->positioned ? 1 : 0;
}

// the checks export and import share, before any device work: arguments, ids in range (and, on import, listed once) and an
// endpointer that is up to date with its handle
int check_record_call(mww_endpointer_t *ep, const std::string &call, const int32_t *h_ids, int n, const void *d_records, bool once) {
    if (n < 0 || (n > 0 && (!h_ids || !d_records))) return refuse(call + "needs n >= 0, and ids and records with n > 0");
    if (reinterpret_cast<uintptr_t>(d_records) % 16 != 0) return refuse(call + "the records must be 16-byte aligned");
    std::vector<uint8_t> listed(once ? (size_t)ep->n_streams : 0, 0);
    for (int i = 0; i < n; ++i) {
        if (h_ids[i] < 0 || h_ids[i] >= ep->n_streams)
            return refuse(call + "stream id " + std::to_string(h_ids[i]) + " out of range [0, " + std::to_string(ep->n_streams) + ")");
        if (once && listed[(size_t)h_ids[i]]++) return refuse(call + "stream id " + std::to_string(h_ids[i]) + " is listed twice");
    }
    long long S = 0;
    int buffered = 0, pending = 0;
    if (int rc = read_counters(ep, &S, &buffered, &pending)) return rc;
    if (S != ep->base_seen || buffered != ep->base_buffered || pending != ep->base_pending)
        return refuse(call + "the endpointer is behind its handle's counters: update the endpointer after the handle's last call");
    return MWW_OK;
}

// a host id list -> d_rec_ids, on st; growing the buffer first waits for the call that may still read it
int stage_record_ids(mww_endpointer_t *ep, const int32_t *h_ids, int n, cudaStream_t st) {
    if ((size_t)n > ep->rec_ids_cap) {
        if (ep->d_rec_ids) { ECU(cudaStreamSynchronize(st)); cudaFree(ep->d_rec_ids); ep->d_rec_ids = nullptr; ep->rec_ids_cap = 0; }
        const size_t want = std::max<size_t>((size_t)n, 1024);
        ECU(cudaMalloc(&ep->d_rec_ids, want * sizeof(int32_t)));
        ep->rec_ids_cap = want;
    }
    ECU(cudaMemcpyAsync(ep->d_rec_ids, h_ids, (size_t)n * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    return MWW_OK;
}

EpRecJob record_job(const mww_endpointer_t *ep) {
    EpRecJob J;
    J.a = ep->a;
    J.base = ep->base_seen;
    J.L = endpoint_record_layout(ep->a.rule.vad_window);
    return J;
}

}  // namespace

extern "C" {

int mww_endpointer_create(const mww_t *h, int model, const mww_endpoint_rule *rule, int capacity, mww_endpointer_t **out) {
    const std::string call = "mww_endpointer_create: ";
    if (!out) return refuse(call + "out is NULL");
    *out = nullptr;
    if (!h) return refuse(call + "needs a handle");
    if (!rule) return refuse(call + "rule is NULL");
    int cap = 0;
    long long seen = 0;
    mww_get_audio_history(h, &cap, &seen);
    if (cap == 0) return refuse(call + "the handle keeps no audio history (mww_set_audio_history)");
    const int K = mww_model_count(h);
    if (K == 0) return refuse(call + "the handle is frontend-only: an endpointer reads a model's probabilities");
    if (model < 0 || model >= K) return refuse(call + "model " + std::to_string(model) + " of a handle of " + std::to_string(K) + " model(s)");
    if (rule->vad_window < 1 || rule->vad_window > kDetectorMaxWindow) return refuse(call + "vad_window must be in [1, 32]");
    if (!std::isfinite(rule->vad_cutoff)) return refuse(call + "vad_cutoff must be finite");
    if (rule->speech_steps < 1 || rule->silence_steps < 1 || rule->timeout_steps < 1 || rule->max_steps < 1)
        return refuse(call + "speech_steps, silence_steps, timeout_steps and max_steps must be at least 1");
    if (rule->lookback_steps < 0 || rule->lookback_steps > kEndpointMaxLookback) return refuse(call + "lookback_steps must be in [0, 64]");
    if (capacity < 1) return refuse(call + "capacity must be at least 1");
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0)
        return fail(nullptr, MWW_ECUDA, std::string("no CUDA device available (this library has no CPU fallback): ") + cudaGetErrorString(e));
    mww_info info, mi;
    mww_get_info(h, &info);
    mww_get_model_info(h, model, &mi);
    mww_endpointer_t *ep = new mww_endpointer;
    ep->h = h; ep->device = info.device; ep->model = model; ep->stride = mi.input_feature_slices; ep->hop = info.hop_samples;
    ep->n_streams = info.n_streams; ep->capacity = capacity;
    ep->members.resize((size_t)mi.n_streams);
    int n_ids = 0;
    mww_get_model_streams(h, model, ep->members.data(), mi.n_streams, &n_ids);
    ep->row_of.assign((size_t)info.n_streams, -1);
    for (int r = 0; r < mi.n_streams; ++r) ep->row_of[ep->members[r]] = r;
    EndpointArgs &a = ep->a;
    a.rule = *rule;
    a.n_rows = mi.n_streams; a.n_streams = info.n_streams; a.capacity = capacity;
    a.step_samples = (long long)ep->stride * ep->hop;
    ep->base_seen = seen; ep->base_buffered = info.frontend_buffered; ep->base_pending = mi.pending_rows;
    DeviceGuard guard(ep->device);
    if (guard.err != cudaSuccess) { delete ep; return cuda_fail(nullptr, guard.err, "cudaSetDevice"); }
    if (int rc = endpointer_alloc(ep)) { endpointer_free(ep); return rc; }
    *out = ep;
    return MWW_OK;
}

int mww_endpointer_destroy(mww_endpointer_t *ep) {
    if (!ep) return MWW_OK;
    DeviceGuard guard(ep->device);
    cudaDeviceSynchronize();
    endpointer_free(ep);
    return MWW_OK;
}

int mww_endpointer_info(const mww_endpointer_t *ep, mww_endpointer_desc *out) {
    if (!ep || !out) return refuse("mww_endpointer_info: needs an endpointer and out");
    *out = mww_endpointer_desc{};
    out->n_rows = ep->a.n_rows; out->model = ep->model; out->stride = ep->stride; out->hop_samples = ep->hop;
    out->capacity = ep->capacity; out->device = ep->device; out->rule = ep->a.rule; out->steps = ep->steps; out->launches = ep->launches;
    return MWW_OK;
}

int mww_endpointer_update(mww_endpointer_t *ep, const float *d_probs, int n, long long pitch, void *cu_stream) {
    const std::string call = "mww_endpointer_update: ";
    if (!ep) return refuse(call + "endpointer is NULL");
    if (n < 0 || pitch < n || (n > 0 && ep->a.n_rows > 0 && !d_probs)) return refuse(call + "needs n >= 0, pitch >= n and probabilities");
    long long S = 0;
    int buffered = 0, pending = 0;
    if (int rc = read_counters(ep, &S, &buffered, &pending)) return rc;
    if (!endpoint_update_fits(ep->base_seen, ep->base_buffered, ep->base_pending, S, buffered, pending, ep->hop, ep->stride, n))
        return refuse(call + std::to_string(n) + " steps do not match the rows the handle emitted since the last update (a skipped update, "
                      "or a full reset of the handle without a reset of the endpointer)");
    DeviceGuard guard(ep->device);
    if (guard.err != cudaSuccess) return cuda_fail(nullptr, guard.err, "cudaSetDevice");
    const long long pos0 = endpoint_position(S, buffered, ep->hop, pending, ep->stride, n, 0);
    if (ep->positioned) ECU(launch_endpoint_update_muted(ep->a, ep->d_mute, d_probs, pitch, n, pos0, static_cast<cudaStream_t>(cu_stream)));
    else ECU(launch_endpoint_update(ep->a, d_probs, pitch, n, pos0, static_cast<cudaStream_t>(cu_stream)));
    ep->launches += 1;
    ep->base_seen = S; ep->base_buffered = buffered; ep->base_pending = pending;
    const int keep = std::min(n, kEndpointMaxLookback);
    for (int i = kEndpointMaxLookback - 1; i >= keep; --i) ep->pos[i] = ep->pos[i - keep];
    for (int i = 0; i < keep; ++i) ep->pos[i] = pos0 + (long long)(n - 1 - i) * ep->a.step_samples;
    ep->steps += n;
    return MWW_OK;
}

int mww_endpointer_arm(mww_endpointer_t *ep, const int32_t *h_ids, int n, void *cu_stream) {
    if (!ep) return refuse("mww_endpointer_arm: endpointer is NULL");
    cudaStream_t st = static_cast<cudaStream_t>(cu_stream);
    DeviceGuard guard(ep->device);
    int m = 0;
    if (int rc = stage_ids(ep, "mww_endpointer_arm", h_ids, n, &m, st)) return rc;
    return arm(ep, ep->d_ids, m, st);
}

int mww_endpointer_arm_device(mww_endpointer_t *ep, const int32_t *d_ids, int n, void *cu_stream) {
    if (!ep) return refuse("mww_endpointer_arm_device: endpointer is NULL");
    if (n < 0 || (n > 0 && !d_ids)) return refuse("mww_endpointer_arm_device: needs n >= 0 and ids with n > 0");
    return arm(ep, d_ids, n, static_cast<cudaStream_t>(cu_stream));
}

int mww_endpointer_disarm(mww_endpointer_t *ep, const int32_t *h_ids, int n, void *cu_stream) {
    if (!ep) return refuse("mww_endpointer_disarm: endpointer is NULL");
    cudaStream_t st = static_cast<cudaStream_t>(cu_stream);
    DeviceGuard guard(ep->device);
    int m = 0;
    if (int rc = stage_ids(ep, "mww_endpointer_disarm", h_ids, n, &m, st)) return rc;
    return clear(ep, ep->d_ids, m, 0, st);
}

int mww_endpointer_reset(mww_endpointer_t *ep, const int32_t *h_ids, int n, void *cu_stream) {
    if (!ep) return refuse("mww_endpointer_reset: endpointer is NULL");
    cudaStream_t st = static_cast<cudaStream_t>(cu_stream);
    DeviceGuard guard(ep->device);
    if (!h_ids) {
        long long S = 0;
        int buffered = 0, pending = 0;
        if (int rc = read_counters(ep, &S, &buffered, &pending)) return rc;
        if (int rc = clear(ep, nullptr, ep->a.n_rows, 1, st)) return rc;
        // a new baseline may be a new axis (mww_reset_frontend, mww_set_audio_history): no replay crosses it
        ep->base_seen = S; ep->base_buffered = buffered; ep->base_pending = pending;
        ep->steps = 0;
        for (long long &p : ep->pos) p = 0;
        return MWW_OK;
    }
    int m = 0;
    if (int rc = stage_ids(ep, "mww_endpointer_reset", h_ids, n, &m, st)) return rc;
    return clear(ep, ep->d_ids, m, 1, st);
}

int mww_endpointer_reset_device(mww_endpointer_t *ep, const int32_t *d_ids, int n, void *cu_stream) {
    if (!ep) return refuse("mww_endpointer_reset_device: endpointer is NULL");
    if (n < 0 || (n > 0 && !d_ids)) return refuse("mww_endpointer_reset_device: needs n >= 0 and ids with n > 0");
    return clear(ep, d_ids, n, 1, static_cast<cudaStream_t>(cu_stream));
}

int mww_endpointer_drain(mww_endpointer_t *ep, mww_endpoint_event *h_events, int max_events, long long *n_events, void *cu_stream) {
    if (!ep) return refuse("mww_endpointer_drain: endpointer is NULL");
    if (max_events < 0 || (max_events > 0 && !h_events)) return refuse("mww_endpointer_drain: needs max_events >= 0 and a buffer");
    DeviceGuard guard(ep->device);
    cudaStream_t st = static_cast<cudaStream_t>(cu_stream);
    ECU(cudaStreamSynchronize(st));
    unsigned long long count = 0;
    ECU(cudaMemcpy(&count, ep->a.count, sizeof(count), cudaMemcpyDeviceToHost));
    const long long take = std::min<long long>(std::min<long long>((long long)count, ep->capacity), max_events);
    if (take > 0) ECU(cudaMemcpy(h_events, ep->a.events, (size_t)take * sizeof(mww_endpoint_event), cudaMemcpyDeviceToHost));
    if (n_events) *n_events = (long long)count;
    ECU(cudaMemsetAsync(ep->a.count, 0, sizeof(unsigned long long), st));
    ECU(cudaMemsetAsync(ep->a.ended, 0xFF, (size_t)ep->capacity * sizeof(int32_t), st));
    ECU(cudaStreamSynchronize(st));
    return MWW_OK;
}

int mww_endpointer_buffers(mww_endpointer_t *ep, const long long **d_count, const mww_endpoint_event **d_events, const int32_t **d_ended,
                           const int32_t **d_armed, int *capacity) {
    if (!ep) return refuse("mww_endpointer_buffers: endpointer is NULL");
    if (d_count) *d_count = reinterpret_cast<const long long *>(ep->a.count);
    if (d_events) *d_events = ep->a.events;
    if (d_ended) *d_ended = ep->a.ended;
    if (d_armed) *d_armed = ep->a.armed;
    if (capacity) *capacity = ep->capacity;
    return MWW_OK;
}

int mww_endpointer_get_state(mww_endpointer_t *ep, mww_endpoint_state *out) {
    if (!ep || !out) return refuse("mww_endpointer_get_state: needs an endpointer and out");
    DeviceGuard guard(ep->device);
    ECU(cudaDeviceSynchronize());
    const EndpointArgs &a = ep->a;
    const size_t R = (size_t)a.n_rows, W = (size_t)(a.rule.vad_window - 1);
    if (out->hist && W > 0) {
        std::vector<float> t(W * R);
        ECU(cudaMemcpy(t.data(), a.hist, t.size() * sizeof(float), cudaMemcpyDeviceToHost));
        for (size_t r = 0; r < R; ++r)
            for (size_t j = 0; j < W; ++j) out->hist[r * W + j] = t[j * R + r];
    }
    if (out->seen) ECU(cudaMemcpy(out->seen, a.seen, R * 8, cudaMemcpyDeviceToHost));
    if (out->flags) ECU(cudaMemcpy(out->flags, a.flags, R * 8, cudaMemcpyDeviceToHost));
    if (out->armed) ECU(cudaMemcpy(out->armed, a.armed, R * 4, cudaMemcpyDeviceToHost));
    if (out->elapsed) ECU(cudaMemcpy(out->elapsed, a.elapsed, R * 4, cudaMemcpyDeviceToHost));
    if (out->run) ECU(cudaMemcpy(out->run, a.run, R * 4, cudaMemcpyDeviceToHost));
    if (out->silence) ECU(cudaMemcpy(out->silence, a.silence, R * 4, cudaMemcpyDeviceToHost));
    if (out->heard) ECU(cudaMemcpy(out->heard, a.heard, R * 4, cudaMemcpyDeviceToHost));
    if (out->start_sample) ECU(cudaMemcpy(out->start_sample, a.start, R * 8, cudaMemcpyDeviceToHost));
    if (out->speech_end_sample) ECU(cudaMemcpy(out->speech_end_sample, a.speech_end, R * 8, cudaMemcpyDeviceToHost));
    out->samples_seen = ep->base_seen; out->buffered = ep->base_buffered; out->pending = ep->base_pending; out->steps = ep->steps;
    for (int i = 0; i < kEndpointMaxLookback; ++i) out->positions[i] = ep->pos[i];
    return MWW_OK;
}

int mww_endpointer_set_state(mww_endpointer_t *ep, const mww_endpoint_state *in) {
    const std::string call = "mww_endpointer_set_state: ";
    if (!ep || !in) return refuse(call + "needs an endpointer and a state");
    const EndpointArgs &a = ep->a;
    const size_t R = (size_t)a.n_rows, W = (size_t)(a.rule.vad_window - 1);
    for (size_t r = 0; r < R; ++r) {
        if (in->seen && in->seen[r] < 0) return refuse(call + "a negative seen");
        if ((in->elapsed && in->elapsed[r] < 0) || (in->run && in->run[r] < 0) || (in->silence && in->silence[r] < 0))
            return refuse(call + "a negative count");
        if (in->heard && in->heard[r] != 0 && in->heard[r] != 1) return refuse(call + "heard must be 0 or 1");
        if (in->armed && in->armed[r] != -1 && in->armed[r] != ep->members[r]) return refuse(call + "armed must be -1 or the row's stream");
    }
    if (in->samples_seen < 0 || in->buffered < 0 || in->buffered >= kWindow || in->pending < 0 || in->pending >= ep->stride || in->steps < 0)
        return refuse(call + "the baseline must be samples_seen >= 0, buffered in [0, 480), pending in [0, stride) and steps >= 0");
    DeviceGuard guard(ep->device);
    ECU(cudaDeviceSynchronize());
    if (in->hist && W > 0) {
        std::vector<float> t(W * R);
        for (size_t r = 0; r < R; ++r)
            for (size_t j = 0; j < W; ++j) t[j * R + r] = in->hist[r * W + j];
        ECU(cudaMemcpy(a.hist, t.data(), t.size() * sizeof(float), cudaMemcpyHostToDevice));
    }
    if (in->seen) ECU(cudaMemcpy(a.seen, in->seen, R * 8, cudaMemcpyHostToDevice));
    if (in->flags) ECU(cudaMemcpy(a.flags, in->flags, R * 8, cudaMemcpyHostToDevice));
    if (in->armed) ECU(cudaMemcpy(a.armed, in->armed, R * 4, cudaMemcpyHostToDevice));
    if (in->elapsed) ECU(cudaMemcpy(a.elapsed, in->elapsed, R * 4, cudaMemcpyHostToDevice));
    if (in->run) ECU(cudaMemcpy(a.run, in->run, R * 4, cudaMemcpyHostToDevice));
    if (in->silence) ECU(cudaMemcpy(a.silence, in->silence, R * 4, cudaMemcpyHostToDevice));
    if (in->heard) ECU(cudaMemcpy(a.heard, in->heard, R * 4, cudaMemcpyHostToDevice));
    if (in->start_sample) ECU(cudaMemcpy(a.start, in->start_sample, R * 8, cudaMemcpyHostToDevice));
    if (in->speech_end_sample) ECU(cudaMemcpy(a.speech_end, in->speech_end_sample, R * 8, cudaMemcpyHostToDevice));
    ep->base_seen = in->samples_seen; ep->base_buffered = (int)in->buffered; ep->base_pending = (int)in->pending; ep->steps = in->steps;
    for (int i = 0; i < kEndpointMaxLookback; ++i) ep->pos[i] = in->positions[i];
    return MWW_OK;
}

int mww_endpointer_arm_at(mww_endpointer_t *ep, const int32_t *h_ids, const int64_t *h_positions, int n, long long skip_samples, void *cu_stream) {
    const std::string call = "mww_endpointer_arm_at";
    if (!ep) return refuse(call + ": endpointer is NULL");
    if (n < 0 || (n > 0 && (!h_ids || !h_positions))) return refuse(call + ": needs n >= 0, and ids and positions with n > 0");
    if (int rc = check_skip(call, skip_samples)) return rc;
    // the list filtered to members, each row once at its latest position, staged in d_ids / d_positions
    std::vector<int32_t> ids;
    std::vector<long long> pos;
    std::vector<int> slot(ep->members.size(), -1);
    for (int i = 0; i < n; ++i) {
        if (h_ids[i] < 0 || h_ids[i] >= ep->n_streams)
            return refuse(call + ": stream id " + std::to_string(h_ids[i]) + " out of range [0, " + std::to_string(ep->n_streams) + ")");
        const int r = ep->row_of[h_ids[i]];
        if (r < 0) continue;
        if (slot[r] < 0) { slot[r] = (int)ids.size(); ids.push_back(h_ids[i]); pos.push_back(h_positions[i]); }
        else pos[slot[r]] = std::max<long long>(pos[slot[r]], h_positions[i]);
    }
    cudaStream_t st = static_cast<cudaStream_t>(cu_stream);
    DeviceGuard guard(ep->device);
    if (guard.err != cudaSuccess) return cuda_fail(nullptr, guard.err, "cudaSetDevice");
    // from pageable memory, as stage_ids: the copies have taken the bytes when cudaMemcpyAsync returns
    if (!ids.empty()) {
        ECU(cudaMemcpyAsync(ep->d_ids, ids.data(), ids.size() * sizeof(int32_t), cudaMemcpyHostToDevice, st));
        ECU(cudaMemcpyAsync(ep->d_positions, pos.data(), pos.size() * sizeof(long long), cudaMemcpyHostToDevice, st));
    }
    return arm_at(ep, ep->d_ids, ep->d_positions, (int)ids.size(), skip_samples, st);
}

int mww_endpointer_arm_at_device(mww_endpointer_t *ep, const int32_t *d_ids, const int64_t *d_positions, int n, long long skip_samples,
                                 void *cu_stream) {
    const std::string call = "mww_endpointer_arm_at_device";
    if (!ep) return refuse(call + ": endpointer is NULL");
    if (n < 0 || (n > 0 && (!d_ids || !d_positions))) return refuse(call + ": needs n >= 0, and ids and positions with n > 0");
    if (int rc = check_skip(call, skip_samples)) return rc;
    return arm_at(ep, d_ids, reinterpret_cast<const long long *>(d_positions), n, skip_samples, static_cast<cudaStream_t>(cu_stream));
}

int mww_endpointer_get_mutes(mww_endpointer_t *ep, int32_t *h_mutes) {
    if (!ep || (!h_mutes && ep->a.n_rows > 0)) return refuse("mww_endpointer_get_mutes: needs an endpointer and a buffer");
    DeviceGuard guard(ep->device);
    ECU(cudaDeviceSynchronize());
    if (ep->a.n_rows > 0) ECU(cudaMemcpy(h_mutes, ep->d_mute, (size_t)ep->a.n_rows * sizeof(int32_t), cudaMemcpyDeviceToHost));
    return MWW_OK;
}

int mww_endpointer_set_mutes(mww_endpointer_t *ep, const int32_t *h_mutes) {
    const std::string call = "mww_endpointer_set_mutes: ";
    if (!ep || (!h_mutes && ep->a.n_rows > 0)) return refuse(call + "needs an endpointer and the mute words");
    for (int r = 0; r < ep->a.n_rows; ++r)
        if (h_mutes[r] < 0 || (h_mutes[r] & kEndpointMuteSteps) > kHistoryMaxCapacity)
            return refuse(call + "a mute word holds a count in [0, 2^22] and the placed bit 2^30");
    DeviceGuard guard(ep->device);
    ECU(cudaDeviceSynchronize());
    if (ep->a.n_rows > 0) ECU(cudaMemcpy(ep->d_mute, h_mutes, (size_t)ep->a.n_rows * sizeof(int32_t), cudaMemcpyHostToDevice));
    ep->positioned = true;
    return MWW_OK;
}

int mww_endpointer_read_commands(mww_endpointer_t *ep, mww_t *h, long long pre, long long post, int max_samples, int16_t *d_out,
                                 long long out_stride, int32_t *d_lengths, void *cu_stream) {
    const std::string call = "mww_endpointer_read_commands: ";
    if (!ep) return refuse(call + "endpointer is NULL");
    if (h != ep->h) return refuse(call + "the handle is not the one the endpointer was created from");
    if (pre < 0 || post < 0) return refuse(call + "pre and post must not be negative");
    if (max_samples < 0 || max_samples > kHistoryMaxCapacity) return refuse(call + "max_samples must be in [0, 2^22]");
    if (out_stride < max_samples) return refuse(call + "out_stride must be at least max_samples");
    if (!d_lengths || (max_samples > 0 && !d_out)) return refuse(call + "NULL output");
    const HistoryRing ring = history_ring(h);
    if (!ring.ring) return refuse(call + "the handle keeps no audio history");
    if (ring.poisoned) return refuse(call + "the handle is poisoned: an earlier staged call failed half-way");
    DeviceGuard guard(ep->device);
    if (guard.err != cudaSuccess) return cuda_fail(nullptr, guard.err, "cudaSetDevice");
    ECU(launch_endpoint_read(ring.ring, ring.capacity, ring.seen, ep->a.count, ep->a.events, ep->capacity, pre, post, max_samples, d_out,
                             out_stride, d_lengths, ring.sm_count, static_cast<cudaStream_t>(cu_stream)));
    ep->launches += 1;
    return MWW_OK;
}

int mww_get_endpointer_layout(const mww_endpointer_t *ep, mww_endpointer_layout *out) {
    if (!ep || !out) return refuse("mww_get_endpointer_layout: needs an endpointer and out");
    fill_layout(ep, out);
    return MWW_OK;
}

int mww_export_endpointer_rows(mww_endpointer_t *ep, const int32_t *h_ids, int n, void *d_records, mww_endpointer_layout *out, void *cu_stream) {
    const std::string call = "mww_export_endpointer_rows: ";
    if (!ep) return refuse(call + "endpointer is NULL");
    if (int rc = check_record_call(ep, call, h_ids, n, d_records, false)) return rc;
    if (out) fill_layout(ep, out);
    if (n == 0) return MWW_OK;
    DeviceGuard guard(ep->device);
    if (guard.err != cudaSuccess) return cuda_fail(nullptr, guard.err, "cudaSetDevice");
    cudaStream_t st = static_cast<cudaStream_t>(cu_stream);
    if (int rc = stage_record_ids(ep, h_ids, n, st)) return rc;
    if (ep->positioned) ECU(launch_pack_endpointer_rows_muted(record_job(ep), ep->d_mute, d_records, ep->d_rec_ids, n, st));
    else ECU(launch_pack_endpointer_rows(record_job(ep), d_records, ep->d_rec_ids, n, st));
    ep->launches += 1;
    return MWW_OK;
}

int mww_import_endpointer_rows(mww_endpointer_t *ep, const int32_t *h_ids, int n, const void *d_records, const mww_endpointer_layout *layout,
                               void *cu_stream) {
    const std::string call = "mww_import_endpointer_rows: ";
    if (!ep) return refuse(call + "endpointer is NULL");
    if (!layout) return refuse(call + "layout is NULL");
    if (int rc = check_record_call(ep, call, h_ids, n, d_records, true)) return rc;
    mww_endpointer_layout mine;
    fill_layout(ep, &mine);
    if (const char *field = endpoint_layout_mismatch(*layout, mine))
        return refuse(call + "the records' " + field + " differs from the endpointer's");
    if (layout->pad != 0 && layout->pad != 1) return refuse(call + "the layout's pad (the positioned flag) must be 0 or 1");
    if (layout->pad == 1) ep->positioned = true;          // the records carry mute words: keep them
    if (n == 0) return MWW_OK;
    DeviceGuard guard(ep->device);
    if (guard.err != cudaSuccess) return cuda_fail(nullptr, guard.err, "cudaSetDevice");
    cudaStream_t st = static_cast<cudaStream_t>(cu_stream);
    if (int rc = stage_record_ids(ep, h_ids, n, st)) return rc;
    if (ep->positioned) ECU(launch_unpack_endpointer_rows_muted(record_job(ep), ep->d_mute, d_records, ep->d_rec_ids, n, st));
    else ECU(launch_unpack_endpointer_rows(record_job(ep), d_records, ep->d_rec_ids, n, st));
    ep->launches += 1;
    return MWW_OK;
}

}  // extern "C"
