// mww_detector_capi.cu -- the extern "C" entry points of the streaming detectors (include/mww.h).  Host code only: rules
// and kernels are in mww_detector.{h,cu}, mww_detector_models.{h,cu} and mww_detector_cutoffs.cu.  A detector is an object
// of its own: no handle knows of it, it reads a handle only through public calls, and its messages go where a failed
// create's go (mww_last_error(NULL)).  Both kinds are row sets: the plain detector one WAKE set whose row index is the
// stream (or its stream_ids entry), a models detector one per model, a row per member of the model's stream set.
#include <algorithm>
#include <string>
#include <vector>

#include "mww_capi.h"
#include "mww_kernels.h"

using namespace mww;

namespace {

// one rule over its rows: role, rule, stride, n_rows and the device state, as the models kernel's descriptor holds them
// (the plain detector's flag is its cooldown), and what only the host keeps
struct RowSet : DetectModel {
    std::vector<int32_t> member_row;    // [n_streams]: the row of each global stream id, -1 for a non-member; empty: id = row
    std::vector<double> cutoffs;        // per-row mode: every row's cutoff, the host copy of d_cutoffs; empty in uniform mode
    double *d_cutoffs = nullptr;
};

}  // namespace

struct mww_detector {
    int device = 0;
    bool multi = false;                 // a models detector (mww_multi_detector_create)
    bool per_row = false;               // per-row mode: every used row set with rows has its cutoffs
    std::vector<RowSet> sets;           // the plain detector's one; a models detector's one per model (an OFF model's unused)
    // the event buffers, the plain detector's row -> stream map, and staging for a host row list (mww_detector_reset)
    unsigned long long *count = nullptr; mww_event *events = nullptr; int32_t *fired = nullptr; int capacity = 0;
    int32_t *d_stream_ids = nullptr;
    int32_t *d_rows = nullptr; size_t rows_cap = 0;
    // the kernels' arguments, filled from the row sets at create and at the switch to per-row mode: the plain detector's
    // `a`; a models detector's `m`, the descriptors d_models holds (which the update's check reads), and d_models_rows
    DetectorArgs a;
    DetectModelsArgs m;
    std::vector<DetectModel> models;
    DetectModel *d_models = nullptr;
    DetectModelRows *d_models_rows = nullptr;
    // event positions (mww_time_detector_events): positions [capacity] beside the events once timed; `updated` is set by every
    // update that launched and cleared by a drain, so that a detector with buffered events cannot be timed; `hop` is a models
    // detector's handle's hop at create
    bool timed = false, updated = false;
    long long *positions = nullptr;
    int hop = kHop;
    // grouped detection (mww_group_detector_events): the kernels' group arguments (g.positions is `positions`), n_groups, and the
    // host copy of every row's (plain) or stream's (models) group
    bool grouped = false;
    int n_groups = 0;
    GroupArgs g;
    std::vector<int32_t> groups;
    // the plain detector's row -> stream map as given at create (empty: stream = row)
    std::vector<int32_t> stream_ids;
    // group arbitration (mww_arbitrate_detector_groups): the source handle whose history every update measures, and the kernels'
    // arguments (ring, seen and capacity are read from src at each update); the largest stream id a row reads
    mww_t *arb_src = nullptr;
    ArbitrationArgs r;
    int arb_max_stream = -1;
};

namespace mww {
const int32_t *detector_event_groups(const mww_detector_t *d) { return d->grouped ? d->g.ev_group : nullptr; }
}  // namespace mww

namespace {

#define DCU(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return cuda_fail(nullptr, e_, #call); } while (0)
#define DENTER(d) DeviceGuard guard_((d)->device); if (guard_.err != cudaSuccess) return cuda_fail(nullptr, guard_.err, "cudaSetDevice")

int refuse(const std::string &msg) { return fail(nullptr, MWW_EINVAL, msg); }

void detector_free(mww_detector_t *d) {
    for (RowSet &s : d->sets) {
        cudaFree(s.hist); cudaFree(s.seen); cudaFree(s.flag); cudaFree(const_cast<int32_t *>(s.inv)); cudaFree(s.d_cutoffs);
    }
    cudaFree(d->count); cudaFree(d->events); cudaFree(d->fired); cudaFree(d->d_stream_ids); cudaFree(d->d_rows);
    cudaFree(d->d_models); cudaFree(d->d_models_rows); cudaFree(d->positions);
    cudaFree(const_cast<int32_t *>(d->g.groups)); cudaFree(d->g.pending); cudaFree(d->g.windows); cudaFree(d->g.ev_group); cudaFree(d->g.ev_candidates);
    cudaFree(d->r.levels); cudaFree(d->r.ev_level);
    delete d;
}

// fresh state for the n listed rows (plain) or global stream ids (models) in device memory, or for all (d_rows == nullptr)
cudaError_t reset_rows(const mww_detector_t *d, const int32_t *d_rows, int n, cudaStream_t st) {
    if (d->multi) return launch_detector_models_reset(d->m, d_rows, d_rows ? n : d->m.n_streams, st);
    return launch_detector_reset(d->a, d_rows, d_rows ? n : d->a.n_rows, st);
}

// the device side of the detector the create described: each used row set's state and inverse map, the event buffers at
// their initial values, the plain detector's stream ids, the kernels' arguments, and every row reset
int detector_alloc(mww_detector_t *d, const int32_t *h_stream_ids) {
    const size_t C = (size_t)d->capacity;
    for (RowSet &s : d->sets) {
        if (s.role == MWW_DETECT_OFF) continue;
        const size_t R = (size_t)s.n_rows, W = (size_t)s.rule.window - 1, S = s.member_row.size();
        DCU(cudaMalloc(&s.hist, std::max<size_t>(W * R, 1) * sizeof(float)));
        DCU(cudaMalloc(&s.seen, std::max<size_t>(R, 1) * sizeof(long long)));
        DCU(cudaMalloc(&s.flag, std::max<size_t>(R, 1) * sizeof(int32_t)));
        if (S) {
            int32_t *d_inv = nullptr;
            DCU(cudaMalloc(&d_inv, S * sizeof(int32_t)));
            s.inv = d_inv;
            DCU(cudaMemcpy(d_inv, s.member_row.data(), S * sizeof(int32_t), cudaMemcpyHostToDevice));
        }
    }
    DCU(cudaMalloc(&d->count, sizeof(unsigned long long)));
    DCU(cudaMalloc(&d->events, C * sizeof(mww_event)));
    DCU(cudaMalloc(&d->fired, C * sizeof(int32_t)));
    DCU(cudaMemset(d->count, 0, sizeof(unsigned long long)));
    DCU(cudaMemset(d->events, 0, C * sizeof(mww_event)));
    DCU(cudaMemset(d->fired, 0xFF, C * sizeof(int32_t)));              // -1 in every slot
    if (d->multi) {
        d->models.assign(d->sets.begin(), d->sets.end());               // each set's descriptor
        DCU(cudaMalloc(&d->d_models, d->models.size() * sizeof(DetectModel)));
        DCU(cudaMemcpy(d->d_models, d->models.data(), d->models.size() * sizeof(DetectModel), cudaMemcpyHostToDevice));
        DetectModelsArgs &m = d->m;
        m.models = d->d_models; m.count = d->count; m.events = d->events; m.fired = d->fired; m.capacity = d->capacity;
    } else {
        const RowSet &s = d->sets[0];
        DetectorArgs &a = d->a;
        if (h_stream_ids) {
            DCU(cudaMalloc(&d->d_stream_ids, (size_t)s.n_rows * sizeof(int32_t)));
            DCU(cudaMemcpy(d->d_stream_ids, h_stream_ids, (size_t)s.n_rows * sizeof(int32_t), cudaMemcpyHostToDevice));
            a.stream_ids = d->d_stream_ids;
        }
        a.rule = s.rule; a.n_rows = s.n_rows; a.hist = s.hist; a.seen = s.seen; a.cooldown = s.flag;
        a.count = d->count; a.events = d->events; a.fired = d->fired; a.capacity = d->capacity;
    }
    DCU(reset_rows(d, nullptr, 0, nullptr));
    DCU(cudaDeviceSynchronize());
    return MWW_OK;
}

// the plain detector, or a refusal naming the call and its models counterpart
int plain_arg(const mww_detector_t *d, const char *call, const char *models_call) {
    if (!d) return refuse(std::string(call) + ": detector is NULL");
    if (d->multi) return refuse(std::string(call) + ": a models detector takes " + models_call);
    return MWW_OK;
}

// a models detector, or a refusal naming the call
int models_arg(const mww_detector_t *d, const char *call) {
    if (!d) return refuse(std::string(call) + ": detector is NULL");
    if (!d->multi) return refuse(std::string(call) + ": not a models detector (mww_multi_detector_create)");
    return MWW_OK;
}

// the row set of model k of a models detector, or a refusal naming the call
int model_arg(mww_detector_t *d, int k, const char *call, RowSet **out) {
    if (int rc = models_arg(d, call)) return rc;
    if (k < 0 || k >= d->m.n_models) return refuse(std::string(call) + ": model index out of range");
    if (d->sets[k].role == MWW_DETECT_OFF) return refuse(std::string(call) + ": model is OFF");
    *out = &d->sets[k];
    return MWW_OK;
}

// a row set's state: history (device [window - 1][n_rows], host [n_rows][window - 1]), seen, and flag (cooldown or active)
int get_state(mww_detector_t *d, const RowSet &s, float *h_hist, long long *h_seen, int32_t *h_flag) {
    DENTER(d);
    DCU(cudaDeviceSynchronize());
    const size_t R = (size_t)s.n_rows, W = (size_t)s.rule.window - 1;
    if (R == 0) return MWW_OK;
    if (h_hist && W) {
        std::vector<float> t(W * R);
        DCU(cudaMemcpy(t.data(), s.hist, W * R * sizeof(float), cudaMemcpyDeviceToHost));
        for (size_t j = 0; j < W; ++j)
            for (size_t r = 0; r < R; ++r) h_hist[r * W + j] = t[j * R + r];
    }
    if (h_seen) DCU(cudaMemcpy(h_seen, s.seen, R * sizeof(long long), cudaMemcpyDeviceToHost));
    if (h_flag) DCU(cudaMemcpy(h_flag, s.flag, R * sizeof(int32_t), cudaMemcpyDeviceToHost));
    return MWW_OK;
}

// the same, written; refused before anything changes unless seen >= 0 and flag in [0, cooldown_slices] (WAKE) or [0, 1] (VAD)
int set_state(mww_detector_t *d, const RowSet &s, const char *call, const float *h_hist, const long long *h_seen, const int32_t *h_flag) {
    const size_t R = (size_t)s.n_rows, W = (size_t)s.rule.window - 1;
    const bool wake = s.role == MWW_DETECT_WAKE;
    const int hi = wake ? s.rule.cooldown_slices : 1;
    for (size_t r = 0; r < R; ++r) {
        if (h_seen && h_seen[r] < 0) return refuse(std::string(call) + ": seen must not be negative");
        if (h_flag && (h_flag[r] < 0 || h_flag[r] > hi))
            return refuse(std::string(call) + (wake ? ": cooldown outside [0, cooldown_slices]" : ": active must be 0 or 1"));
    }
    DENTER(d);
    DCU(cudaDeviceSynchronize());
    if (R == 0) return MWW_OK;
    if (h_hist && W) {
        std::vector<float> t(W * R);
        for (size_t j = 0; j < W; ++j)
            for (size_t r = 0; r < R; ++r) t[j * R + r] = h_hist[r * W + j];
        DCU(cudaMemcpy(s.hist, t.data(), W * R * sizeof(float), cudaMemcpyHostToDevice));
    }
    if (h_seen) DCU(cudaMemcpy(s.seen, h_seen, R * sizeof(long long), cudaMemcpyHostToDevice));
    if (h_flag) DCU(cudaMemcpy(s.flag, h_flag, R * sizeof(int32_t), cudaMemcpyHostToDevice));
    return MWW_OK;
}

// The detector to per-row mode: every row of every used row set at its rule's cutoff, on the device too, and a models
// detector's descriptors that carry those arrays.  On a failure nothing is kept and the detector stays in uniform mode.
int to_row_cutoffs(mww_detector_t *d, cudaStream_t st) {
    auto undo = [&](cudaError_t e, const char *what) {
        for (RowSet &s : d->sets) { cudaFree(s.d_cutoffs); s.d_cutoffs = nullptr; s.cutoffs.clear(); }
        cudaFree(d->d_models_rows); d->d_models_rows = nullptr;
        return cuda_fail(nullptr, e, what);
    };
    for (RowSet &s : d->sets) {
        if (s.role == MWW_DETECT_OFF || s.n_rows == 0) continue;
        s.cutoffs.assign((size_t)s.n_rows, s.rule.cutoff);
        double *p = nullptr;
        if (cudaError_t e = cudaMalloc(&p, s.cutoffs.size() * sizeof(double))) return undo(e, "cudaMalloc");
        s.d_cutoffs = p;
        if (cudaError_t e = cudaMemcpyAsync(p, s.cutoffs.data(), s.cutoffs.size() * sizeof(double), cudaMemcpyHostToDevice, st))
            return undo(e, "cudaMemcpyAsync");
    }
    if (d->multi) {
        std::vector<DetectModelRows> rows(d->models.size());
        for (size_t k = 0; k < rows.size(); ++k) rows[k] = {d->models[k], d->sets[k].d_cutoffs};
        DetectModelRows *p = nullptr;
        if (cudaError_t e = cudaMalloc(&p, rows.size() * sizeof(DetectModelRows))) return undo(e, "cudaMalloc");
        d->d_models_rows = p;
        if (cudaError_t e = cudaMemcpyAsync(p, rows.data(), rows.size() * sizeof(DetectModelRows), cudaMemcpyHostToDevice, st))
            return undo(e, "cudaMemcpyAsync");
    }
    d->per_row = true;
    return MWW_OK;
}

// The listed ids' cutoffs in row set s (ids are rows, or global stream ids where the set has a member map), checked
// before anything changes: finite cutoffs, ids in range, each naming a row, none twice.  The first call with an id
// switches the detector to per-row mode; then the span of rows the call touched is copied on cu_stream.
int set_cutoffs(mww_detector_t *d, RowSet &s, const std::string &call, const char *ids_name, const int32_t *h_ids, const double *h_cutoffs,
                int n, void *cu_stream) {
    if (n < 0) return refuse(call + ": n must not be negative");
    if (n == 0) return MWW_OK;
    if (!h_ids || !h_cutoffs) return refuse(call + ": " + ids_name + " and h_cutoffs must not be NULL");
    const bool by_stream = !s.member_row.empty();
    const int n_ids = by_stream ? (int)s.member_row.size() : s.n_rows;
    std::vector<char> listed((size_t)std::max(s.n_rows, 1), 0);
    std::vector<int32_t> rows((size_t)n);
    int lo = s.n_rows, hi = -1;
    for (int i = 0; i < n; ++i) {
        if (!(h_cutoffs[i] - h_cutoffs[i] == 0.0)) return refuse(call + ": cutoffs must be finite");
        const int32_t id = h_ids[i];
        if (id < 0 || id >= n_ids) return refuse(call + ": id " + std::to_string(id) + " out of range");
        const int32_t r = by_stream ? s.member_row[id] : id;
        if (r < 0) return refuse(call + ": stream " + std::to_string(id) + " is not a member of the model's stream set");
        if (listed[r]) return refuse(call + ": id " + std::to_string(id) + " listed twice");
        listed[r] = 1;
        rows[i] = r;
        lo = std::min(lo, (int)r); hi = std::max(hi, (int)r);
    }
    DENTER(d);
    cudaStream_t st = static_cast<cudaStream_t>(cu_stream);
    if (!d->per_row) {
        if (int rc = to_row_cutoffs(d, st)) return rc;
    }
    for (int i = 0; i < n; ++i) s.cutoffs[rows[i]] = h_cutoffs[i];
    // from pageable memory: the call returns once the span is staged, so later changes to the host copy cannot reach it
    DCU(cudaMemcpyAsync(s.d_cutoffs + lo, s.cutoffs.data() + lo, (size_t)(hi - lo + 1) * sizeof(double), cudaMemcpyHostToDevice, st));
    return MWW_OK;
}

// every row's cutoff: the rule's in uniform mode
void get_cutoffs(const mww_detector_t *d, const RowSet &s, double *h_cutoffs) {
    for (int r = 0; r < s.n_rows; ++r) h_cutoffs[r] = d->per_row ? s.cutoffs[r] : s.rule.cutoff;
}

// n ids from host memory into the staging buffer d_rows, on st; growing the buffer first waits for the call that may still
// read it
int stage_ids(mww_detector_t *d, const int32_t *h_ids, int n, cudaStream_t st) {
    if ((size_t)n > d->rows_cap) {
        if (d->d_rows) { DCU(cudaStreamSynchronize(st)); cudaFree(d->d_rows); d->d_rows = nullptr; d->rows_cap = 0; }
        const size_t want = std::max<size_t>((size_t)n, 1024);
        DCU(cudaMalloc(&d->d_rows, want * sizeof(int32_t)));
        d->rows_cap = want;
    }
    DCU(cudaMemcpyAsync(d->d_rows, h_ids, (size_t)n * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    return MWW_OK;
}

// one models update call's description, checked as mww_multi_detector_update checks it; *any: some model has work
int models_call(const mww_detector_t *d, const std::string &name, const float *const *d_probs, const long long *pitch, const int *n_steps,
                const int *pending_before, DetectCall *call, bool *any) {
    if (!d_probs || !pitch || !n_steps || !pending_before) return refuse(name + ": d_probs, pitch, n_steps and pending_before must not be NULL");
    *any = false;
    for (int k = 0; k < d->m.n_models; ++k) {
        const DetectModel &M = d->models[k];
        if (M.role == MWW_DETECT_OFF) continue;
        DetectCall &c = call[k];
        c.probs = d_probs[k]; c.pitch = pitch[k]; c.n_steps = n_steps[k]; c.pending = pending_before[k];
        if (c.n_steps > 0 && M.n_rows > 0) {
            if (!c.probs || c.pitch < c.n_steps)
                return refuse(name + ": model " + std::to_string(k) + " needs d_probs and n_steps columns within the row pitch");
            *any = true;
        }
    }
    if (!detect_call_fits(d->models.data(), call, d->m.n_models))
        return refuse(name + ": the step counts and pending rows do not describe one call "
                      "(n_k = (p_k + R) div s_k with 0 <= p_k < s_k for one R >= 0)");
    return MWW_OK;
}

// ---- detector records: each row set is one model of the record (the plain detector's one WAKE model, row = id)
void fill_layout(const mww_detector_t *d, mww_detector_layout *o) {
    *o = mww_detector_layout{};
    o->multi = d->multi ? 1 : 0;
    o->n_models = (int32_t)d->sets.size();
    for (size_t k = 0; k < d->sets.size(); ++k) {
        const RowSet &s = d->sets[k];
        o->role[k] = s.role;
        if (s.role == MWW_DETECT_OFF) continue;
        o->window[k] = s.rule.window;
        o->cooldown_slices[k] = s.role == MWW_DETECT_WAKE ? s.rule.cooldown_slices : 0;
    }
    const std::vector<DetectModel> models(d->sets.begin(), d->sets.end());
    o->record_bytes = detector_record_layout(models.data(), o->n_models).record_bytes;
}

DetRecJob record_job(const mww_detector_t *d) {
    const std::vector<DetectModel> models(d->sets.begin(), d->sets.end());
    return detector_record_job(models.data(), (int)models.size());
}

// the checks both calls make before any device work: n, the records buffer, ids in range (rows of a plain detector,
// global stream ids of a models detector) and, on import, listed once
int check_rows(const mww_detector_t *d, const std::string &call, const int32_t *h_ids, int n, const void *d_records, bool once) {
    if (n < 0) return refuse(call + ": n must not be negative");
    if (n == 0) return MWW_OK;
    if (!h_ids) return refuse(call + ": h_ids is NULL");
    if (!d_records || reinterpret_cast<uintptr_t>(d_records) % 16) return refuse(call + ": d_records must be a 16-byte aligned device buffer");
    const int n_ids = d->multi ? d->m.n_streams : d->sets[0].n_rows;
    std::vector<char> listed(once ? (size_t)n_ids : 0, 0);
    for (int i = 0; i < n; ++i) {
        const int32_t id = h_ids[i];
        if (id < 0 || id >= n_ids) return refuse(call + ": id " + std::to_string(id) + " out of range");
        if (once) {
            if (listed[id]) return refuse(call + ": id " + std::to_string(id) + " listed twice");
            listed[id] = 1;
        }
    }
    return MWW_OK;
}

// The drains: the events (and, h_positions != nullptr, their positions; h_groups != nullptr, their groups and candidates) to the
// host; the counter cleared, d_fired and a timed detector's positions refilled with -1
int drain(mww_detector_t *d, mww_event *h_events, long long *h_positions, int max_events, long long *n_events, cudaStream_t st,
          int32_t *h_groups = nullptr, int32_t *h_candidates = nullptr, float *h_levels = nullptr) {
    DENTER(d);
    unsigned long long count = 0;
    DCU(cudaMemcpyAsync(&count, d->count, sizeof(count), cudaMemcpyDeviceToHost, st));
    DCU(cudaStreamSynchronize(st));
    const size_t stored = (size_t)std::min<unsigned long long>(count, (unsigned long long)d->capacity);
    const size_t n = std::min(stored, (size_t)max_events);
    if (n) DCU(cudaMemcpyAsync(h_events, d->events, n * sizeof(mww_event), cudaMemcpyDeviceToHost, st));
    if (n && h_positions) DCU(cudaMemcpyAsync(h_positions, d->positions, n * sizeof(long long), cudaMemcpyDeviceToHost, st));
    if (n && h_groups) {
        DCU(cudaMemcpyAsync(h_groups, d->g.ev_group, n * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
        DCU(cudaMemcpyAsync(h_candidates, d->g.ev_candidates, n * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    }
    if (n && h_levels) DCU(cudaMemcpyAsync(h_levels, d->r.ev_level, n * sizeof(float), cudaMemcpyDeviceToHost, st));
    if (stored) {
        DCU(cudaMemsetAsync(d->count, 0, sizeof(count), st));
        DCU(cudaMemsetAsync(d->fired, 0xFF, stored * sizeof(int32_t), st));
        if (d->timed) DCU(cudaMemsetAsync(d->positions, 0xFF, stored * sizeof(long long), st));
    }
    if (n) DCU(cudaStreamSynchronize(st));
    *n_events = (long long)count;
    d->updated = false;
    return MWW_OK;
}

// the untimed update calls refuse a timed detector, the timed ones an untimed detector
int untimed_arg(const mww_detector_t *d, const char *call, const char *timed_call) {
    if (d->timed) return refuse(std::string(call) + ": the detector is timed (mww_time_detector_events): it takes " + timed_call);
    return MWW_OK;
}
int timed_arg(const mww_detector_t *d, const char *call) {
    if (!d->timed) return refuse(std::string(call) + ": the detector is not timed: call mww_time_detector_events after create or a drain");
    return MWW_OK;
}

// ---- grouped detection
int grouped_arg(const mww_detector_t *d, const std::string &call) {
    if (!d) return refuse(call + ": detector is NULL");
    if (!d->grouped) return refuse(call + ": the detector is not grouped (mww_group_detector_events)");
    return MWW_OK;
}

// ids a grouped detector keys groups by: rows (plain) or global stream ids (models); its group slots
int group_ids(const mww_detector_t *d) { return d->multi ? d->m.n_streams : d->sets[0].n_rows; }
int group_slots(const mww_detector_t *d) { return d->g.n_slots; }

// the listed ids' groups, checked before anything changes: ids in range and listed once, groups in [-1, n_groups); then the
// span of ids the call touched is copied on cu_stream
int set_groups(mww_detector_t *d, const std::string &call, const int32_t *h_ids, const int32_t *h_groups, int n, void *cu_stream) {
    if (int rc = grouped_arg(d, call)) return rc;
    if (n < 0) return refuse(call + ": n must not be negative");
    if (n == 0) return MWW_OK;
    if (!h_ids || !h_groups) return refuse(call + ": ids and h_groups must not be NULL");
    const int n_ids = group_ids(d);
    std::vector<char> listed((size_t)n_ids, 0);
    int lo = n_ids, hi = -1;
    for (int i = 0; i < n; ++i) {
        const int32_t id = h_ids[i], grp = h_groups[i];
        if (id < 0 || id >= n_ids) return refuse(call + ": id " + std::to_string(id) + " out of range");
        if (listed[id]) return refuse(call + ": id " + std::to_string(id) + " listed twice");
        if (grp < -1 || grp >= d->n_groups) return refuse(call + ": group " + std::to_string(grp) + " outside [-1, n_groups)");
        listed[id] = 1;
        lo = std::min(lo, (int)id); hi = std::max(hi, (int)id);
    }
    DENTER(d);
    for (int i = 0; i < n; ++i) d->groups[h_ids[i]] = h_groups[i];
    // from pageable memory: the call returns once the span is staged
    DCU(cudaMemcpyAsync(const_cast<int32_t *>(d->g.groups) + lo, d->groups.data() + lo, (size_t)(hi - lo + 1) * sizeof(int32_t), cudaMemcpyHostToDevice,
                        static_cast<cudaStream_t>(cu_stream)));
    return MWW_OK;
}

// ---- group arbitration
int arbitrated_arg(const mww_detector_t *d, const std::string &call) {
    if (int rc = grouped_arg(d, call)) return rc;
    if (!d->arb_src) return refuse(call + ": the detector is not arbitrated (mww_arbitrate_detector_groups)");
    return MWW_OK;
}

// an arbitrated update's source history, read now and checked: src healthy, still holding Ls + Ln samples and every stream a
// row reads
int arbitration_clock(mww_detector_t *d, const std::string &call) {
    const HistoryRing h = history_ring(d->arb_src);
    if (h.poisoned) return refuse(call + ": the arbitration source handle failed a staged call and cannot be read");
    if (h.capacity < d->r.speech + d->r.noise)
        return refuse(call + ": the arbitration source keeps " + std::to_string(h.capacity) + " samples of audio history; the detector reads " +
                      std::to_string(d->r.speech + d->r.noise) + " (speech_samples + noise_samples)");
    if (d->arb_max_stream >= h.n_streams) return refuse(call + ": a row reads a stream the arbitration source no longer has");
    d->r.ring = h.ring; d->r.capacity = h.capacity; d->r.seen = h.seen;
    return MWW_OK;
}

}  // namespace

extern "C" {

// ---- both kinds
int mww_detector_destroy(mww_detector_t *d) {
    if (!d) return MWW_OK;
    DENTER(d);
    cudaDeviceSynchronize();
    detector_free(d);
    return MWW_OK;
}

int mww_detector_drain(mww_detector_t *d, mww_event *h_events, int max_events, long long *n_events, void *cu_stream) {
    if (!d || !n_events || max_events < 0 || (max_events > 0 && !h_events))
        return refuse("mww_detector_drain: needs a detector, n_events and room for max_events >= 0 events");
    return drain(d, h_events, nullptr, max_events, n_events, static_cast<cudaStream_t>(cu_stream));
}

int mww_detector_buffers(mww_detector_t *d, const long long **d_count, const mww_event **d_events, const int32_t **d_fired, int *capacity) {
    if (!d) return refuse("mww_detector_buffers: detector is NULL");
    if (d_count) *d_count = reinterpret_cast<const long long *>(d->count);
    if (d_events) *d_events = d->events;
    if (d_fired) *d_fired = d->fired;
    if (capacity) *capacity = d->capacity;
    return MWW_OK;
}

int mww_detector_reset_device(mww_detector_t *d, const int32_t *d_rows, int n, void *cu_stream) {
    if (!d || n < 0) return refuse("mww_detector_reset_device: needs a detector and n >= 0");
    DENTER(d);
    DCU(reset_rows(d, d_rows, n, static_cast<cudaStream_t>(cu_stream)));
    return MWW_OK;
}

int mww_detector_reset(mww_detector_t *d, const int32_t *h_rows, int n, void *cu_stream) {
    if (!d || n < 0) return refuse("mww_detector_reset: needs a detector and n >= 0");
    if (!h_rows) return mww_detector_reset_device(d, nullptr, 0, cu_stream);
    if (n == 0) return MWW_OK;
    DENTER(d);
    cudaStream_t st = static_cast<cudaStream_t>(cu_stream);
    if (int rc = stage_ids(d, h_rows, n, st)) return rc;
    DCU(reset_rows(d, d->d_rows, n, st));
    return MWW_OK;
}

// ---- detector records, both kinds
int mww_get_detector_layout(const mww_detector_t *d, mww_detector_layout *out) {
    if (!d || !out) return refuse("mww_get_detector_layout: needs a detector and out");
    fill_layout(d, out);
    return MWW_OK;
}

int mww_export_detector_rows(mww_detector_t *d, const int32_t *h_ids, int n, void *d_records, mww_detector_layout *out, void *cu_stream) {
    const std::string call = "mww_export_detector_rows";
    if (!d) return refuse(call + ": detector is NULL");
    if (int rc = check_rows(d, call, h_ids, n, d_records, false)) return rc;
    if (out) fill_layout(d, out);
    if (n == 0) return MWW_OK;
    DENTER(d);
    cudaStream_t st = static_cast<cudaStream_t>(cu_stream);
    if (int rc = stage_ids(d, h_ids, n, st)) return rc;
    DCU(launch_pack_detector_rows(record_job(d), d_records, d->d_rows, n, st));
    return MWW_OK;
}

int mww_import_detector_rows(mww_detector_t *d, const int32_t *h_ids, int n, const void *d_records, const mww_detector_layout *layout,
                             void *cu_stream) {
    const std::string call = "mww_import_detector_rows";
    if (!d || !layout) return refuse(call + ": needs a detector and the records' layout");
    mww_detector_layout mine;
    fill_layout(d, &mine);
    int which = -1;
    if (const char *field = detector_layout_mismatch(*layout, mine, &which))
        return refuse(call + ": the records do not fit this detector: " + field + (which >= 0 ? " of model " + std::to_string(which) : std::string()) +
                      " differs");
    if (int rc = check_rows(d, call, h_ids, n, d_records, true)) return rc;
    if (n == 0) return MWW_OK;
    DENTER(d);
    cudaStream_t st = static_cast<cudaStream_t>(cu_stream);
    if (int rc = stage_ids(d, h_ids, n, st)) return rc;
    DCU(launch_unpack_detector_rows(record_job(d), d_records, d->d_rows, n, st));
    return MWW_OK;
}

// ---- the plain detector: row set 0
int mww_detector_create(int device, int n_rows, int window, double cutoff, int cooldown_slices, int capacity,
                        const int32_t *h_stream_ids, mww_detector_t **out) {
    if (!out) return refuse("mww_detector_create: out is NULL");
    *out = nullptr;
    if (n_rows < 1) return refuse("mww_detector_create: n_rows must be at least 1");
    if (window < 1 || window > kDetectorMaxWindow) return refuse("mww_detector_create: window must be in [1, 32]");
    if (!(cutoff - cutoff == 0.0)) return refuse("mww_detector_create: cutoff must be finite");
    if (cooldown_slices < 0) return refuse("mww_detector_create: cooldown_slices must not be negative");
    if (capacity < 1) return refuse("mww_detector_create: capacity must be at least 1");
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0)
        return fail(nullptr, MWW_ECUDA, std::string("no CUDA device available (this library has no CPU fallback): ") + cudaGetErrorString(e));
    if (device < 0 || device >= count) return refuse("mww_detector_create: device index out of range");
    DeviceGuard guard(device);
    if (guard.err != cudaSuccess) return cuda_fail(nullptr, guard.err, "cudaSetDevice");
    mww_detector_t *d = new mww_detector;
    d->device = device;
    d->capacity = capacity;
    RowSet &s = d->sets.emplace_back();
    s.role = MWW_DETECT_WAKE;
    s.rule.window = window; s.rule.cutoff = cutoff; s.rule.cooldown_slices = cooldown_slices;
    s.n_rows = n_rows;
    if (h_stream_ids) d->stream_ids.assign(h_stream_ids, h_stream_ids + n_rows);
    if (int rc = detector_alloc(d, h_stream_ids)) { detector_free(d); return rc; }
    *out = d;
    return MWW_OK;
}

int mww_detector_update(mww_detector_t *d, const float *d_probs, int n_steps, long long pitch, void *cu_stream) {
    if (int rc = plain_arg(d, "mww_detector_update", "mww_multi_detector_update")) return rc;
    if (int rc = untimed_arg(d, "mww_detector_update", "mww_update_detector_at")) return rc;
    if (n_steps < 0 || (n_steps > 0 && (!d_probs || pitch < n_steps)))
        return refuse("mww_detector_update: needs d_probs and n_steps >= 0 columns within the row pitch");
    if (n_steps == 0) return MWW_OK;
    DENTER(d);
    if (d->per_row) DCU(launch_detector_update_cutoffs(d->a, d->sets[0].d_cutoffs, d_probs, n_steps, pitch, static_cast<cudaStream_t>(cu_stream)));
    else DCU(launch_detector_update(d->a, d_probs, n_steps, pitch, static_cast<cudaStream_t>(cu_stream)));
    d->updated = true;
    return MWW_OK;
}

int mww_detector_get_state(mww_detector_t *d, float *h_hist, long long *h_seen, int32_t *h_cooldown) {
    if (int rc = plain_arg(d, "mww_detector_get_state", "mww_multi_detector_get_state")) return rc;
    return get_state(d, d->sets[0], h_hist, h_seen, h_cooldown);
}

int mww_detector_set_state(mww_detector_t *d, const float *h_hist, const long long *h_seen, const int32_t *h_cooldown) {
    if (int rc = plain_arg(d, "mww_detector_set_state", "mww_multi_detector_set_state")) return rc;
    return set_state(d, d->sets[0], "mww_detector_set_state", h_hist, h_seen, h_cooldown);
}

int mww_set_detector_cutoffs(mww_detector_t *d, const int32_t *h_rows, const double *h_cutoffs, int n, void *cu_stream) {
    if (int rc = plain_arg(d, "mww_set_detector_cutoffs", "mww_set_multi_detector_cutoffs")) return rc;
    return set_cutoffs(d, d->sets[0], "mww_set_detector_cutoffs", "h_rows", h_rows, h_cutoffs, n, cu_stream);
}

int mww_get_detector_cutoffs(mww_detector_t *d, double *h_cutoffs) {
    if (!d || !h_cutoffs) return refuse("mww_get_detector_cutoffs: needs a detector and h_cutoffs");
    if (int rc = plain_arg(d, "mww_get_detector_cutoffs", "mww_get_multi_detector_cutoffs")) return rc;
    get_cutoffs(d, d->sets[0], h_cutoffs);
    return MWW_OK;
}

// ---- the models detector: a row set per model
int mww_multi_detector_create(const mww_t *h, const mww_detect_rule *rules, int capacity, mww_detector_t **out) {
    const std::string call = "mww_multi_detector_create: ";
    if (!out) return refuse(call + "out is NULL");
    *out = nullptr;
    if (!rules) return refuse(call + "rules is NULL");
    if (capacity < 1) return refuse(call + "capacity must be at least 1");
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0)
        return fail(nullptr, MWW_ECUDA, std::string("no CUDA device available (this library has no CPU fallback): ") + cudaGetErrorString(e));
    if (!h) return refuse(call + "handle is NULL");
    const int K = mww_model_count(h);
    if (K < 1) return refuse(call + "the handle is frontend-only: it has no models to detect with");
    int n_wake = 0, vad = -1;
    for (int k = 0; k < K; ++k) {
        const mww_detect_rule &r = rules[k];
        const std::string at = call + "model " + std::to_string(k) + ": ";
        if (r.role != MWW_DETECT_OFF && r.role != MWW_DETECT_WAKE && r.role != MWW_DETECT_VAD)
            return refuse(at + "role must be MWW_DETECT_OFF, _WAKE or _VAD");
        if (r.role == MWW_DETECT_OFF) continue;
        if (r.window < 1 || r.window > kDetectorMaxWindow) return refuse(at + "window must be in [1, 32]");
        if (!(r.cutoff - r.cutoff == 0.0)) return refuse(at + "cutoff must be finite");
        if (r.role == MWW_DETECT_WAKE && r.cooldown_slices < 0) return refuse(at + "cooldown_slices must not be negative");
        if (r.role == MWW_DETECT_WAKE) ++n_wake;
        if (r.role == MWW_DETECT_VAD) {
            if (vad >= 0) return refuse(call + "at most one model may be the VAD");
            vad = k;
        }
    }
    if (n_wake == 0) return refuse(call + "at least one model must be WAKE");
    mww_info info;
    if (mww_get_info(h, &info) != MWW_OK) return refuse(call + "cannot read the handle");
    mww_detector_t *d = new mww_detector;
    d->device = info.device;
    d->multi = true;
    d->capacity = capacity;
    d->hop = info.hop_samples;
    d->sets.resize(K);
    DetectModelsArgs &m = d->m;
    m.n_streams = info.n_streams; m.n_models = K; m.vad = vad;
    std::vector<int32_t> ids;
    for (int k = 0; k < K; ++k) {
        const mww_detect_rule &r = rules[k];
        RowSet &s = d->sets[k];
        s.role = r.role;
        if (r.role == MWW_DETECT_OFF) continue;
        mww_info mi;
        int n = 0;
        if (mww_get_model_info(h, k, &mi) != MWW_OK || mww_get_model_streams(h, k, nullptr, 0, &n) != MWW_OK) { delete d; return refuse(call + "cannot read a model"); }
        ids.resize((size_t)n);
        if (n > 0 && mww_get_model_streams(h, k, ids.data(), n, &n) != MWW_OK) { delete d; return refuse(call + "cannot read a stream set"); }
        s.rule.window = r.window; s.rule.cutoff = r.cutoff; s.rule.cooldown_slices = r.role == MWW_DETECT_WAKE ? r.cooldown_slices : 0;
        s.stride = std::max(mi.input_feature_slices, 1);
        s.n_rows = n;
        if (n != m.n_streams) {                 // a stream set is all streams exactly when it has every id: then row = stream
            s.member_row.assign((size_t)m.n_streams, -1);
            for (int i = 0; i < n; ++i) s.member_row[ids[i]] = i;
        }
        if (r.role == MWW_DETECT_WAKE) m.wake[m.n_wake++] = (int8_t)k;
    }
    DeviceGuard guard(d->device);
    if (guard.err != cudaSuccess) { delete d; return cuda_fail(nullptr, guard.err, "cudaSetDevice"); }
    if (int rc = detector_alloc(d, nullptr)) { detector_free(d); return rc; }
    *out = d;
    return MWW_OK;
}

int mww_multi_detector_update(mww_detector_t *d, const float *const *d_probs, const long long *pitch, const int *n_steps,
                               const int *pending_before, void *cu_stream) {
    if (int rc = models_arg(d, "mww_multi_detector_update")) return rc;
    if (int rc = untimed_arg(d, "mww_multi_detector_update", "mww_update_multi_detector_at")) return rc;
    DetectModelsArgs &m = d->m;
    DetectCall call[kDetectMaxModels];
    bool any = false;
    if (int rc = models_call(d, "mww_multi_detector_update", d_probs, pitch, n_steps, pending_before, call, &any)) return rc;
    if (!any) return MWW_OK;
    DENTER(d);
    for (int k = 0; k < m.n_models; ++k) m.call[k] = call[k];
    if (d->per_row) DCU(launch_detector_models_update_cutoffs(detect_args_rows(m, d->d_models_rows), static_cast<cudaStream_t>(cu_stream)));
    else DCU(launch_detector_models_update(m, static_cast<cudaStream_t>(cu_stream)));
    d->updated = true;
    return MWW_OK;
}

int mww_multi_detector_get_state(mww_detector_t *d, int k, float *h_hist, long long *h_seen, int32_t *h_cooldown_or_active) {
    RowSet *s = nullptr;
    if (int rc = model_arg(d, k, "mww_multi_detector_get_state", &s)) return rc;
    return get_state(d, *s, h_hist, h_seen, h_cooldown_or_active);
}

int mww_multi_detector_set_state(mww_detector_t *d, int k, const float *h_hist, const long long *h_seen, const int32_t *h_cooldown_or_active) {
    RowSet *s = nullptr;
    if (int rc = model_arg(d, k, "mww_multi_detector_set_state", &s)) return rc;
    return set_state(d, *s, "mww_multi_detector_set_state", h_hist, h_seen, h_cooldown_or_active);
}

int mww_set_multi_detector_cutoffs(mww_detector_t *d, int k, const int32_t *h_stream_ids, const double *h_cutoffs, int n, void *cu_stream) {
    RowSet *s = nullptr;
    if (int rc = model_arg(d, k, "mww_set_multi_detector_cutoffs", &s)) return rc;
    return set_cutoffs(d, *s, "mww_set_multi_detector_cutoffs", "h_stream_ids", h_stream_ids, h_cutoffs, n, cu_stream);
}

int mww_get_multi_detector_cutoffs(mww_detector_t *d, int k, double *h_cutoffs) {
    RowSet *s = nullptr;
    if (int rc = model_arg(d, k, "mww_get_multi_detector_cutoffs", &s)) return rc;
    if (!h_cutoffs && s->n_rows > 0) return refuse("mww_get_multi_detector_cutoffs: h_cutoffs is NULL");
    get_cutoffs(d, *s, h_cutoffs);
    return MWW_OK;
}

// ---- event positions (both kinds)
int mww_time_detector_events(mww_detector_t *d) {
    const std::string call = "mww_time_detector_events";
    if (!d) return refuse(call + ": detector is NULL");
    if (d->timed) return MWW_OK;
    if (d->updated) return refuse(call + ": the detector may hold events: time it after create or a drain, before any update");
    DENTER(d);
    long long *p = nullptr;
    DCU(cudaMalloc(&p, (size_t)d->capacity * sizeof(long long)));
    if (cudaError_t e = cudaMemset(p, 0xFF, (size_t)d->capacity * sizeof(long long))) { cudaFree(p); return cuda_fail(nullptr, e, "cudaMemset"); }
    d->positions = p;
    d->timed = true;
    return MWW_OK;
}

int mww_update_detector_at(mww_detector_t *d, const float *d_probs, int n_steps, long long pitch, long long last_end, long long step_samples,
                           void *cu_stream) {
    const char *call = "mww_update_detector_at";
    if (int rc = plain_arg(d, call, "mww_update_multi_detector_at")) return rc;
    if (int rc = timed_arg(d, call)) return rc;
    if (n_steps < 0 || (n_steps > 0 && (!d_probs || pitch < n_steps)))
        return refuse(std::string(call) + ": needs d_probs and n_steps >= 0 columns within the row pitch");
    if (step_samples < 1) return refuse(std::string(call) + ": step_samples must be at least 1");
    if (n_steps == 0) return MWW_OK;
    DENTER(d);
    const double *cut = d->per_row ? d->sets[0].d_cutoffs : nullptr;
    if (d->arb_src) {
        if (int rc = arbitration_clock(d, call)) return rc;
        DCU(launch_detector_update_arbitrated(d->a, cut, d_probs, n_steps, pitch, d->g, d->r, last_end, step_samples, static_cast<cudaStream_t>(cu_stream)));
    } else if (d->grouped) DCU(launch_detector_update_grouped(d->a, cut, d_probs, n_steps, pitch, d->g, last_end, step_samples, static_cast<cudaStream_t>(cu_stream)));
    else DCU(launch_detector_update_at(d->a, cut, d_probs, n_steps, pitch, d->positions, last_end, step_samples, static_cast<cudaStream_t>(cu_stream)));
    d->updated = true;
    return MWW_OK;
}

int mww_update_multi_detector_at(mww_detector_t *d, const float *const *d_probs, const long long *pitch, const int *n_steps,
                                 const int *pending_before, const int *pending_after, long long row_end, void *cu_stream) {
    const std::string call = "mww_update_multi_detector_at";
    if (int rc = models_arg(d, call.c_str())) return rc;
    if (int rc = timed_arg(d, call.c_str())) return rc;
    DetectModelsArgs &m = d->m;
    DetectCall c[kDetectMaxModels];
    bool any = false;
    if (int rc = models_call(d, call, d_probs, pitch, n_steps, pending_before, c, &any)) return rc;
    if (!pending_after) return refuse(call + ": pending_after must not be NULL");
    const long long R = event_call_rows(d->models.data(), c, pending_after, m.n_models);
    if (R < 0)
        return refuse(call + ": the step counts and pending rows before and after do not describe one call "
                      "(R = n_k s_k - p_k + g_k with 0 <= p_k, g_k < s_k, the same R >= 0 for every model)");
    // a grouped detector closes its windows at every call that moved the clock, even one in which no model ran a step
    if (!any && !(d->grouped && R > 0)) return MWW_OK;
    if (d->arb_src)
        if (int rc = arbitration_clock(d, call)) return rc;
    DENTER(d);
    for (int k = 0; k < m.n_models; ++k) m.call[k] = c[k];
    const long long row0 = event_row0_end(row_end, d->hop, R);
    cudaStream_t st = static_cast<cudaStream_t>(cu_stream);
    if (d->arb_src) {
        if (d->per_row) DCU(launch_detector_models_update_arbitrated(detect_args_rows(m, d->d_models_rows), m, d->g, d->r, row0, row_end, d->hop, st));
        else DCU(launch_detector_models_update_arbitrated(m, d->g, d->r, row0, row_end, d->hop, st));
    } else if (d->grouped) {
        if (d->per_row) DCU(launch_detector_models_update_grouped(detect_args_rows(m, d->d_models_rows), m, d->g, row0, row_end, d->hop, st));
        else DCU(launch_detector_models_update_grouped(m, d->g, row0, row_end, d->hop, st));
    } else if (d->per_row) {
        DCU(launch_detector_models_update_at(detect_args_rows(m, d->d_models_rows), d->positions, row0, d->hop, st));
    } else {
        DCU(launch_detector_models_update_at(m, d->positions, row0, d->hop, st));
    }
    d->updated = true;
    return MWW_OK;
}

int mww_get_detector_positions(mww_detector_t *d, const int64_t **d_positions) {
    if (!d || !d_positions) return refuse("mww_get_detector_positions: needs a detector and d_positions");
    if (int rc = timed_arg(d, "mww_get_detector_positions")) return rc;
    *d_positions = reinterpret_cast<const int64_t *>(d->positions);
    return MWW_OK;
}

int mww_drain_detector_at(mww_detector_t *d, mww_event *h_events, int64_t *h_positions, int max_events, long long *n_events, void *cu_stream) {
    if (!d || !n_events || max_events < 0 || (max_events > 0 && (!h_events || !h_positions)))
        return refuse("mww_drain_detector_at: needs a detector, n_events and room for max_events >= 0 events and positions");
    if (int rc = timed_arg(d, "mww_drain_detector_at")) return rc;
    return drain(d, h_events, reinterpret_cast<long long *>(h_positions), max_events, n_events, static_cast<cudaStream_t>(cu_stream));
}

// ---- grouped detection (both kinds)
int mww_group_detector_events(mww_detector_t *d, int n_groups, long long window_samples) {
    const std::string call = "mww_group_detector_events";
    if (!d) return refuse(call + ": detector is NULL");
    if (!d->timed) return refuse(call + ": only a timed detector can be grouped (mww_time_detector_events)");
    if (d->grouped) return refuse(call + ": the detector is already grouped");
    if (d->updated) return refuse(call + ": the detector may hold events: group it after create or a drain, before any update");
    const int n_ids = group_ids(d);
    if (n_groups < 1 || n_groups > n_ids)
        return refuse(call + ": n_groups must be in [1, " + std::to_string(n_ids) + (d->multi ? "] (n_streams)" : "] (n_rows)"));
    if (window_samples < 0 || window_samples > (1LL << 22)) return refuse(call + ": window_samples must be in [0, 2^22]");
    DENTER(d);
    GroupArgs g;
    g.positions = d->positions;
    g.window = window_samples;
    g.n_wake = d->multi ? d->m.n_wake : 1;
    g.n_slots = n_groups * g.n_wake;
    for (int w = 0; w < g.n_wake && d->multi; ++w) g.wake_of[d->m.wake[w]] = (int8_t)w;
    auto undo = [&](cudaError_t e, const char *what) {
        cudaFree(const_cast<int32_t *>(g.groups)); cudaFree(g.pending); cudaFree(g.windows); cudaFree(g.ev_group); cudaFree(g.ev_candidates);
        return cuda_fail(nullptr, e, what);
    };
    const size_t S = (size_t)g.n_slots, C = (size_t)d->capacity;
    int32_t *groups = nullptr;
    if (cudaError_t e = cudaMalloc(&groups, (size_t)n_ids * sizeof(int32_t))) return undo(e, "cudaMalloc");
    g.groups = groups;
    if (cudaError_t e = cudaMalloc(&g.pending, S * sizeof(GroupPending))) return undo(e, "cudaMalloc");
    if (cudaError_t e = cudaMalloc(&g.windows, S * sizeof(mww_group_window))) return undo(e, "cudaMalloc");
    if (cudaError_t e = cudaMalloc(&g.ev_group, C * sizeof(int32_t))) return undo(e, "cudaMalloc");
    if (cudaError_t e = cudaMalloc(&g.ev_candidates, C * sizeof(int32_t))) return undo(e, "cudaMalloc");
    const std::vector<GroupPending> pending(S);
    if (cudaError_t e = cudaMemset(groups, 0xFF, (size_t)n_ids * sizeof(int32_t))) return undo(e, "cudaMemset");
    if (cudaError_t e = cudaMemcpy(g.pending, pending.data(), S * sizeof(GroupPending), cudaMemcpyHostToDevice)) return undo(e, "cudaMemcpy");
    if (cudaError_t e = cudaMemset(g.windows, 0, S * sizeof(mww_group_window))) return undo(e, "cudaMemset");
    d->g = g;
    d->groups.assign((size_t)n_ids, -1);
    d->n_groups = n_groups;
    d->grouped = true;
    return MWW_OK;
}

int mww_set_detector_groups(mww_detector_t *d, const int32_t *h_rows, const int32_t *h_groups, int n, void *cu_stream) {
    if (int rc = plain_arg(d, "mww_set_detector_groups", "mww_set_multi_detector_groups")) return rc;
    return set_groups(d, "mww_set_detector_groups", h_rows, h_groups, n, cu_stream);
}

int mww_set_multi_detector_groups(mww_detector_t *d, const int32_t *h_stream_ids, const int32_t *h_groups, int n, void *cu_stream) {
    if (int rc = models_arg(d, "mww_set_multi_detector_groups")) return rc;
    return set_groups(d, "mww_set_multi_detector_groups", h_stream_ids, h_groups, n, cu_stream);
}

int mww_get_detector_groups(mww_detector_t *d, int32_t *h_groups) {
    if (int rc = plain_arg(d, "mww_get_detector_groups", "mww_get_multi_detector_groups")) return rc;
    if (int rc = grouped_arg(d, "mww_get_detector_groups")) return rc;
    if (!h_groups) return refuse("mww_get_detector_groups: h_groups is NULL");
    std::copy(d->groups.begin(), d->groups.end(), h_groups);
    return MWW_OK;
}

int mww_get_multi_detector_groups(mww_detector_t *d, int32_t *h_groups) {
    if (int rc = models_arg(d, "mww_get_multi_detector_groups")) return rc;
    if (int rc = grouped_arg(d, "mww_get_multi_detector_groups")) return rc;
    if (!h_groups) return refuse("mww_get_multi_detector_groups: h_groups is NULL");
    std::copy(d->groups.begin(), d->groups.end(), h_groups);
    return MWW_OK;
}

int mww_flush_detector_groups(mww_detector_t *d, void *cu_stream) {
    if (int rc = grouped_arg(d, "mww_flush_detector_groups")) return rc;
    DENTER(d);
    cudaStream_t st = static_cast<cudaStream_t>(cu_stream);
    if (d->arb_src && d->multi) DCU(launch_detector_models_arbitrated_flush(d->m, d->g, d->r, st));
    else if (d->arb_src) DCU(launch_detector_arbitrated_flush(d->a, d->g, d->r, st));
    else if (d->multi) DCU(launch_detector_models_groups_flush(d->m, d->g, st));
    else DCU(launch_detector_groups_flush(d->a, d->g, st));
    d->updated = true;
    return MWW_OK;
}

int mww_drain_detector_groups(mww_detector_t *d, mww_event *h_events, int64_t *h_positions, int32_t *h_groups, int32_t *h_candidates,
                              int max_events, long long *n_events, void *cu_stream) {
    if (!d || !n_events || max_events < 0 || (max_events > 0 && (!h_events || !h_positions || !h_groups || !h_candidates)))
        return refuse("mww_drain_detector_groups: needs a detector, n_events and room for max_events >= 0 events, positions, groups and "
                      "candidates");
    if (int rc = grouped_arg(d, "mww_drain_detector_groups")) return rc;
    return drain(d, h_events, reinterpret_cast<long long *>(h_positions), max_events, n_events, static_cast<cudaStream_t>(cu_stream), h_groups,
                 h_candidates);
}

int mww_get_detector_group_windows(mww_detector_t *d, mww_group_window *h_windows) {
    if (int rc = grouped_arg(d, "mww_get_detector_group_windows")) return rc;
    if (!h_windows) return refuse("mww_get_detector_group_windows: h_windows is NULL");
    DENTER(d);
    DCU(cudaDeviceSynchronize());
    DCU(cudaMemcpy(h_windows, d->g.windows, (size_t)group_slots(d) * sizeof(mww_group_window), cudaMemcpyDeviceToHost));
    return MWW_OK;
}

int mww_set_detector_group_windows(mww_detector_t *d, const mww_group_window *h_windows) {
    const std::string call = "mww_set_detector_group_windows";
    if (int rc = grouped_arg(d, call)) return rc;
    if (!h_windows) return refuse(call + ": h_windows is NULL");
    for (int s = 0; s < group_slots(d); ++s) {
        const mww_group_window &w = h_windows[s];
        if (w.open != 0 && w.open != 1) return refuse(call + ": slot " + std::to_string(s) + ": open must be 0 or 1");
        if (w.open && w.candidates < 1) return refuse(call + ": slot " + std::to_string(s) + ": an open window needs candidates >= 1");
    }
    DENTER(d);
    DCU(cudaDeviceSynchronize());
    DCU(cudaMemcpy(d->g.windows, h_windows, (size_t)group_slots(d) * sizeof(mww_group_window), cudaMemcpyHostToDevice));
    return MWW_OK;
}

// ---- group arbitration (both kinds)
int mww_arbitrate_detector_groups(mww_detector_t *d, mww_t *src, int speech_samples, int noise_samples) {
    const std::string call = "mww_arbitrate_detector_groups";
    if (int rc = grouped_arg(d, call)) return rc;
    if (d->arb_src) return refuse(call + ": the detector is already arbitrated");
    if (d->updated) return refuse(call + ": the detector may hold events: arbitrate it after grouping or a drain, before any update");
    if (!src) return refuse(call + ": src is NULL");
    mww_info info;
    if (mww_get_info(src, &info) != MWW_OK) return refuse(call + ": cannot read the source handle");
    if (info.device != d->device) return refuse(call + ": the source handle is on another device than the detector");
    const HistoryRing h = history_ring(src);
    if (h.poisoned) return refuse(call + ": the source handle failed a staged call and cannot be read");
    const std::string range = "[" + std::to_string(kArbitrationMinSamples) + ", 2^20]";
    if (speech_samples < kArbitrationMinSamples || speech_samples > kArbitrationMaxSamples) return refuse(call + ": speech_samples must be in " + range);
    if (noise_samples < kArbitrationMinSamples || noise_samples > kArbitrationMaxSamples) return refuse(call + ": noise_samples must be in " + range);
    if ((long long)speech_samples + noise_samples > h.capacity)
        return refuse(call + ": speech_samples + noise_samples (" + std::to_string((long long)speech_samples + noise_samples) +
                      ") exceed the source's audio history (" + std::to_string(h.capacity) + " samples)");
    int lo = 0, hi = 0;
    if (d->multi) {
        hi = d->m.n_streams - 1;
    } else if (!d->stream_ids.empty()) {
        lo = *std::min_element(d->stream_ids.begin(), d->stream_ids.end());
        hi = *std::max_element(d->stream_ids.begin(), d->stream_ids.end());
    } else {
        hi = d->sets[0].n_rows - 1;
    }
    if (lo < 0 || hi >= info.n_streams)
        return refuse(call + ": the rows read streams in [" + std::to_string(lo) + ", " + std::to_string(hi) + "]; the source has " +
                      std::to_string(info.n_streams));
    DENTER(d);
    ArbitrationArgs r;
    r.speech = speech_samples; r.noise = noise_samples;
    const size_t S = (size_t)group_slots(d), C = (size_t)d->capacity;
    auto undo = [&](cudaError_t e, const char *what) { cudaFree(r.levels); cudaFree(r.ev_level); return cuda_fail(nullptr, e, what); };
    if (cudaError_t e = cudaMalloc(&r.levels, S * sizeof(float))) return undo(e, "cudaMalloc");
    if (cudaError_t e = cudaMalloc(&r.ev_level, C * sizeof(float))) return undo(e, "cudaMalloc");
    if (cudaError_t e = cudaMemset(r.levels, 0, S * sizeof(float))) return undo(e, "cudaMemset");
    d->r = r;
    d->arb_src = src;
    d->arb_max_stream = hi;
    return MWW_OK;
}

int mww_drain_detector_arbitrated(mww_detector_t *d, mww_event *h_events, int64_t *h_positions, int32_t *h_groups, int32_t *h_candidates,
                                  float *h_levels, int max_events, long long *n_events, void *cu_stream) {
    if (!d || !n_events || max_events < 0 || (max_events > 0 && (!h_events || !h_positions || !h_groups || !h_candidates || !h_levels)))
        return refuse("mww_drain_detector_arbitrated: needs a detector, n_events and room for max_events >= 0 events, positions, groups, "
                      "candidates and levels");
    if (int rc = arbitrated_arg(d, "mww_drain_detector_arbitrated")) return rc;
    return drain(d, h_events, reinterpret_cast<long long *>(h_positions), max_events, n_events, static_cast<cudaStream_t>(cu_stream), h_groups,
                 h_candidates, h_levels);
}

int mww_get_detector_group_levels(mww_detector_t *d, float *h_levels) {
    if (int rc = arbitrated_arg(d, "mww_get_detector_group_levels")) return rc;
    if (!h_levels) return refuse("mww_get_detector_group_levels: h_levels is NULL");
    DENTER(d);
    DCU(cudaDeviceSynchronize());
    DCU(cudaMemcpy(h_levels, d->r.levels, (size_t)group_slots(d) * sizeof(float), cudaMemcpyDeviceToHost));
    return MWW_OK;
}

int mww_set_detector_group_levels(mww_detector_t *d, const float *h_levels) {
    const std::string call = "mww_set_detector_group_levels";
    if (int rc = arbitrated_arg(d, call)) return rc;
    if (!h_levels) return refuse(call + ": h_levels is NULL");
    for (int s = 0; s < group_slots(d); ++s)
        if (!(h_levels[s] >= 0.f && h_levels[s] <= 3.4028234663852886e38f))
            return refuse(call + ": slot " + std::to_string(s) + ": a level must be finite and not negative");
    DENTER(d);
    DCU(cudaDeviceSynchronize());
    DCU(cudaMemcpy(d->r.levels, h_levels, (size_t)group_slots(d) * sizeof(float), cudaMemcpyHostToDevice));
    return MWW_OK;
}

}  // extern "C"
