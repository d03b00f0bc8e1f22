// tests/emul_detector_models.cc -- TEST INFRASTRUCTURE: the multi-model detector's per-stream body and reset
// (microwakeword_b200/csrc/mww_detector_models.h) run on the CPU, stream by stream as the kernel's threads run them, lanes
// past the last stream of the last warp included, for tests/test_detector_models.py.  Host state has the device layout:
// hist [window - 1][n_rows], seen [n_rows], flag [n_rows] per model.
#include <vector>

#include "../microwakeword_b200/csrc/mww_detector_models.h"

using namespace mww;

namespace {

struct Sink {                // what the kernel's ballot and atomicAdd do, one event at a time
    mww_event *events; int capacity; long long count; int32_t *fired;
    void operator()(bool fire, int k, int stream, long long step, float score) {
        if (!fire) return;
        if (count < capacity) { events[count] = mww_event{stream, k, step, score, 0}; fired[count] = stream; }
        ++count;
    }
};

// the create's descriptors and the call's parameters, from flat per-model arrays (inv[k] == NULL: all streams)
void make_args(int n_streams, int K, const int *roles, const int *windows, const int *cooldowns, const double *cutoffs,
               const int *strides, const int *n_rows, int32_t *const *inv, float *const *hist, long long *const *seen,
               int32_t *const *flag, std::vector<DetectModel> &models, DetectModelsArgs &a) {
    models.assign(K, DetectModel());
    a.n_streams = n_streams; a.n_models = K; a.vad = -1; a.n_wake = 0;
    for (int k = 0; k < K; ++k) {
        DetectModel &M = models[k];
        M.role = roles[k];
        M.rule.window = windows[k]; M.rule.cutoff = cutoffs[k]; M.rule.cooldown_slices = cooldowns[k];
        M.stride = strides[k]; M.n_rows = n_rows[k];
        M.inv = inv[k]; M.hist = hist[k]; M.seen = seen[k]; M.flag = flag[k];
        if (M.role == MWW_DETECT_VAD) a.vad = k;
        if (M.role == MWW_DETECT_WAKE) a.wake[a.n_wake++] = (int8_t)k;
    }
    a.models = models.data();
}

}  // namespace

extern "C" {

int emul_sizeof_rule() { return (int)sizeof(mww_detect_rule); }

// detect_call_fits on the given roles, strides, step counts and pending rows
int emul_call_fits(int K, const int *roles, const int *strides, const int *n_steps, const int *pending) {
    std::vector<DetectModel> models(K);
    std::vector<DetectCall> call(K);
    for (int k = 0; k < K; ++k) {
        models[k].role = roles[k]; models[k].stride = strides[k];
        call[k].n_steps = n_steps[k]; call[k].pending = pending[k];
    }
    return detect_call_fits(models.data(), call.data(), K) ? 1 : 0;
}

// one update call.  Events go to events[0, capacity) (fired[] beside them) in the order the streams emit them; returns how
// many fired, -1 when the call does not fit (nothing run)
long long emul_models_update(int n_streams, int K, const int *roles, const int *windows, const int *cooldowns, const double *cutoffs,
                             const int *strides, const int *n_rows, int32_t *const *inv, float *const *hist, long long *const *seen,
                             int32_t *const *flag, const float *const *probs, const long long *pitch, const int *n_steps,
                             const int *pending, mww_event *events, int32_t *fired, int capacity) {
    std::vector<DetectModel> models;
    DetectModelsArgs a;
    make_args(n_streams, K, roles, windows, cooldowns, cutoffs, strides, n_rows, inv, hist, seen, flag, models, a);
    for (int k = 0; k < K; ++k) {
        a.call[k].probs = probs[k]; a.call[k].pitch = pitch[k]; a.call[k].n_steps = n_steps[k]; a.call[k].pending = pending[k];
    }
    if (!detect_call_fits(models.data(), a.call, K)) return -1;
    a.capacity = capacity;
    Sink sink{events, capacity, 0, fired};
    const int lanes = (n_streams + 31) / 32 * 32;
    for (int s = 0; s < lanes; ++s) detect_models_stream(a, s, sink);
    return sink.count;
}

// the reset kernel's body over ids[0, n) or, ids == NULL, streams [0, n_streams)
void emul_models_reset(int n_streams, int K, const int *roles, const int *windows, const int *cooldowns, const double *cutoffs,
                       const int *strides, const int *n_rows, int32_t *const *inv, float *const *hist, long long *const *seen,
                       int32_t *const *flag, const int32_t *ids, int n) {
    std::vector<DetectModel> models;
    DetectModelsArgs a;
    make_args(n_streams, K, roles, windows, cooldowns, cutoffs, strides, n_rows, inv, hist, seen, flag, models, a);
    if (!ids) n = n_streams;
    for (int i = 0; i < n; ++i) detect_models_reset_stream(a, ids ? ids[i] : i);
}

}  // extern "C"
