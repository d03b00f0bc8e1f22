// tests/emul_detector_cutoffs.cc -- TEST INFRASTRUCTURE: both detectors in per-row mode, on the CPU: the plain detector's
// rule (microwakeword_b200/csrc/mww_detector.h) in the thread and warp forms of detector_update_kernel<*, true>, each row
// compared against its own cutoff, and the models detector's per-stream body and reset
// (microwakeword_b200/csrc/mww_detector_models.h) over per-row descriptors, for tests/test_detector_cutoffs.py.  Host state
// has the layouts of tests/emul_detector.cc (plain: hist [n_rows][window - 1]) and tests/emul_detector_models.cc (models:
// the device layout).
#include <vector>

#include "../microwakeword_b200/csrc/mww_detector_models.h"

using namespace mww;

namespace {

struct RowHistory {          // host state is [n_rows][window - 1]: a row's entries are contiguous
    float *h;
    float get(int j) const { return h[j]; }
    void set(int j, float v) { h[j] = v; }
};

struct PassWindow {          // what the kernel's shuffles read: the lanes' registers of this pass and the one before
    const float *cur, *prev;
    float operator()(int i) const { return i >= 0 ? cur[i & 31] : prev[i & 31]; }
};

struct Sink {
    mww_event *events; int max; long long count;
    void add(int row, long long step, float score) {
        if (count < max) events[count] = mww_event{row, 0, step, score, 0};
        ++count;
    }
};

struct ModelSink {           // what the kernel's ballot and atomicAdd do, one event at a time
    mww_event *events; int capacity; long long count; int32_t *fired;
    void operator()(bool fire, int k, int stream, long long step, float score) {
        if (!fire) return;
        if (count < capacity) { events[count] = mww_event{stream, k, step, score, 0}; fired[count] = stream; }
        ++count;
    }
};

DetectorRule rule(int window, int cooldown_slices) {
    DetectorRule r;
    r.window = window; r.cooldown_slices = cooldown_slices; r.cutoff = 0.0;      // per-row mode never reads it
    return r;
}

// per-row descriptors and the call's arguments from flat per-model arrays (inv[k] == NULL: all streams)
void make_args(int n_streams, int K, const int *roles, const int *windows, const int *cooldowns, const double *cutoffs,
               const double *const *row_cutoff, const int *strides, const int *n_rows, int32_t *const *inv, float *const *hist,
               long long *const *seen, int32_t *const *flag, std::vector<DetectModelRows> &models, DetectModelsArgsT<DetectModelRows> &a) {
    models.assign(K, DetectModelRows());
    a.n_streams = n_streams; a.n_models = K; a.vad = -1; a.n_wake = 0;
    for (int k = 0; k < K; ++k) {
        DetectModelRows &M = models[k];
        M.role = roles[k];
        M.rule.window = windows[k]; M.rule.cutoff = cutoffs[k]; M.rule.cooldown_slices = cooldowns[k];
        M.stride = strides[k]; M.n_rows = n_rows[k];
        M.inv = inv[k]; M.hist = hist[k]; M.seen = seen[k]; M.flag = flag[k];
        M.row_cutoff = row_cutoff[k];
        if (M.role == MWW_DETECT_VAD) a.vad = k;
        if (M.role == MWW_DETECT_WAKE) a.wake[a.n_wake++] = (int8_t)k;
    }
    a.models = models.data();
}

}  // namespace

extern "C" {

// one update call of a per-row plain detector, thread form, on host state hist [R][window - 1], seen [R], cooldown [R];
// probs [R][pitch]; row r compared against cutoffs[r].  Events (stream = row) in row-major order of (row, step).
long long emul_rows_update_thread(int window, int cooldown_slices, const double *cutoffs, float *hist, long long *seen, int32_t *cooldown,
                                  const float *probs, int R, int n_steps, long long pitch, mww_event *events, int max_events) {
    const DetectorRule r = rule(window, cooldown_slices);
    Sink out{events, max_events, 0};
    for (int row = 0; row < R; ++row) {
        RowHistory h{hist + (long long)row * (window - 1)};
        const double c = cutoffs[row];           // loaded once per call
        int cd = cooldown[row];
        for (int t = 0; t < n_steps; ++t) {
            float score = 0.f;
            if (detector_step_at(h, r, c, seen[row], cd, probs[row * pitch + t], &score)) out.add(row, seen[row], score);
            ++seen[row];
        }
        cooldown[row] = cd;
    }
    return out.count;
}

// the same call as the warp form runs it: 32-step passes, one average per lane, the ballot against the row's cutoff, the
// chain over the candidate mask
long long emul_rows_update_warp(int window, int cooldown_slices, const double *cutoffs, float *hist, long long *seen, int32_t *cooldown,
                                const float *probs, int R, int n_steps, long long pitch, mww_event *events, int max_events) {
    const DetectorRule r = rule(window, cooldown_slices);
    const int w = window;
    Sink out{events, max_events, 0};
    if (n_steps <= 0) return 0;
    for (int row = 0; row < R; ++row) {
        float *h = hist + (long long)row * (w - 1);
        const float *p = probs + row * pitch;
        const double c = cutoffs[row];
        float cur[32] = {0}, prev[32] = {0};
        for (int lane = 32 - (w - 1); lane < 32; ++lane) prev[lane] = h[lane - (32 - (w - 1))];
        int cd = cooldown[row], n = 0;
        for (int base = 0; base < n_steps; base += 32) {
            n = n_steps - base < 32 ? n_steps - base : 32;
            for (int lane = 0; lane < 32; ++lane) cur[lane] = lane < n ? p[base + lane] : 0.f;
            const PassWindow x{cur, prev};
            const int first = detector_first_full(seen[row] + base, w, n);
            float avg[32];
            unsigned candidates = 0;
            for (int lane = 0; lane < 32; ++lane) {
                avg[lane] = detector_window_mean(x, lane, w);
                if (lane >= first && lane < n && (double)avg[lane] > c) candidates |= 1u << lane;
            }
            const unsigned fired = detector_chain_pass(r, candidates, first, n, cd);
            for (int lane = 0; lane < 32; ++lane)
                if ((fired >> lane) & 1u) out.add(row, seen[row] + base + lane, avg[lane]);
            if (base + 32 < n_steps)
                for (int lane = 0; lane < 32; ++lane) prev[lane] = cur[lane];
        }
        const PassWindow x{cur, prev};
        float keep[32];
        for (int lane = 0; lane < w - 1; ++lane) keep[lane] = x(n - (w - 1) + lane);
        for (int lane = 0; lane < w - 1; ++lane) h[lane] = keep[lane];
        seen[row] += n_steps;
        cooldown[row] = cd;
    }
    return out.count;
}

// one update call of a per-row models detector (row_cutoff[k]: model k's [n_k] cutoffs).  Events go to events[0, capacity)
// (fired[] beside them) in the order the streams emit them; returns how many fired, -1 when the call does not fit
long long emul_rows_models_update(int n_streams, int K, const int *roles, const int *windows, const int *cooldowns, const double *cutoffs,
                                  const double *const *row_cutoff, const int *strides, const int *n_rows, int32_t *const *inv,
                                  float *const *hist, long long *const *seen, int32_t *const *flag, const float *const *probs,
                                  const long long *pitch, const int *n_steps, const int *pending, mww_event *events, int32_t *fired,
                                  int capacity) {
    std::vector<DetectModelRows> models;
    DetectModelsArgsT<DetectModelRows> a;
    make_args(n_streams, K, roles, windows, cooldowns, cutoffs, row_cutoff, strides, n_rows, inv, hist, seen, flag, models, a);
    for (int k = 0; k < K; ++k) {
        a.call[k].probs = probs[k]; a.call[k].pitch = pitch[k]; a.call[k].n_steps = n_steps[k]; a.call[k].pending = pending[k];
    }
    std::vector<DetectModel> plain(models.begin(), models.end());
    if (!detect_call_fits(plain.data(), a.call, K)) return -1;
    a.capacity = capacity;
    ModelSink sink{events, capacity, 0, fired};
    const int lanes = (n_streams + 31) / 32 * 32;
    for (int s = 0; s < lanes; ++s) detect_models_stream(a, s, sink);
    return sink.count;
}

// the reset kernel's body (which runs on plain descriptors in either mode and never touches a cutoff) over ids[0, n) or,
// ids == NULL, streams [0, n_streams)
void emul_rows_models_reset(int n_streams, int K, const int *roles, const int *windows, const int *cooldowns, const double *cutoffs,
                            const double *const *row_cutoff, const int *strides, const int *n_rows, int32_t *const *inv,
                            float *const *hist, long long *const *seen, int32_t *const *flag, const int32_t *ids, int n) {
    std::vector<DetectModelRows> models;
    DetectModelsArgsT<DetectModelRows> rows;
    make_args(n_streams, K, roles, windows, cooldowns, cutoffs, row_cutoff, strides, n_rows, inv, hist, seen, flag, models, rows);
    std::vector<DetectModel> plain(models.begin(), models.end());
    DetectModelsArgs a;
    a.n_streams = n_streams; a.n_models = K; a.models = plain.data();
    if (!ids) n = n_streams;
    for (int i = 0; i < n; ++i) detect_models_reset_stream(a, ids ? ids[i] : i);
}

}  // extern "C"
