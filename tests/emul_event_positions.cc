// tests/emul_event_positions.cc -- TEST INFRASTRUCTURE: the timed detectors' update bodies, the history read that ends at
// given positions and the verifier slots that end at their events (microwakeword_b200/csrc/mww_event_positions.h, with the
// detectors' rule functions of mww_detector.h and mww_detector_models.h) run on the CPU as the kernels of
// mww_event_positions.cu run them -- lane by lane for the warp form, stream by stream for the models body -- for
// tests/test_event_positions.py.  Host detector state has the layouts of tests/emul_detector.cc and
// tests/emul_detector_models.cc.
#include <vector>

#include "../microwakeword_b200/csrc/mww_event_positions.h"

using namespace mww;

namespace {

struct RowHistory {
    float *h;
    float get(int j) const { return h[j]; }
    void set(int j, float v) { h[j] = v; }
};

struct PassWindow {
    const float *cur, *prev;
    float operator()(int i) const { return i >= 0 ? cur[i & 31] : prev[i & 31]; }
};

// events and their positions, as append_events with StepPositions stores them
struct Sink {
    mww_event *events; long long *positions; int max; long long count;
    void add(int row, long long step, float score, long long pos) {
        if (count < max) { events[count] = mww_event{row, 0, step, score, 0}; positions[count] = pos; }
        ++count;
    }
};

DetectorRule rule(int window, double cutoff, int cooldown_slices) {
    DetectorRule r;
    r.window = window; r.cutoff = cutoff; r.cooldown_slices = cooldown_slices;
    return r;
}

// the models kernel's TimedEmit, one event at a time
struct ModelsSink {
    const DetectModelsArgs &a;
    mww_event *events; long long *positions; int capacity; long long count;
    long long row0_end; int hop;
    void operator()(bool fire, int k, int stream, long long step, float score, int j) {
        if (!fire) return;
        if (count < capacity) {
            events[count] = mww_event{stream, k, step, score, 0};
            positions[count] = event_model_step_end(row0_end, hop, j, a.models[k].stride, a.call[k].pending);
        }
        ++count;
    }
};

}  // namespace

extern "C" {

// the thread form: every row's steps in order, step t of the call at event_step_end(last_end, step_samples, n, t)
long long emul_timed_thread(int window, double cutoff, int cooldown_slices, float *hist, long long *seen, int32_t *cooldown, const float *probs,
                            int R, int n_steps, long long pitch, long long last_end, long long step_samples, mww_event *events,
                            long long *positions, int max_events) {
    const DetectorRule r = rule(window, cutoff, cooldown_slices);
    Sink out{events, positions, max_events, 0};
    for (int row = 0; row < R; ++row) {
        RowHistory h{hist + (long long)row * (window - 1)};
        int cd = cooldown[row];
        for (int t = 0; t < n_steps; ++t) {
            float score = 0.f;
            if (detector_step_at(h, r, r.cutoff, seen[row], cd, probs[row * pitch + t], &score))
                out.add(row, seen[row], score, event_step_end(last_end, step_samples, n_steps, t));
            ++seen[row];
        }
        cooldown[row] = cd;
    }
    return out.count;
}

// the warp form, lane by lane: the event of lane `lane` of the pass at `base` is step base + lane of the call
long long emul_timed_warp(int window, double cutoff, int cooldown_slices, float *hist, long long *seen, int32_t *cooldown, const float *probs,
                          int R, int n_steps, long long pitch, long long last_end, long long step_samples, mww_event *events,
                          long long *positions, int max_events) {
    const DetectorRule r = rule(window, cutoff, cooldown_slices);
    const int w = window;
    Sink out{events, positions, max_events, 0};
    if (n_steps <= 0) return 0;
    for (int row = 0; row < R; ++row) {
        float *h = hist + (long long)row * (w - 1);
        const float *p = probs + row * pitch;
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
                if (lane >= first && lane < n && (double)avg[lane] > r.cutoff) candidates |= 1u << lane;
            }
            const unsigned fired = detector_chain_pass(r, candidates, first, n, cd);
            for (int lane = 0; lane < 32; ++lane)
                if ((fired >> lane) & 1u)
                    out.add(row, seen[row] + base + lane, avg[lane], event_step_end(last_end, step_samples, n_steps, base + lane));
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

// event_call_rows on flat per-model arrays
long long emul_call_rows(int K, const int *roles, const int *strides, const int *n_steps, const int *pending, const int *pending_after) {
    std::vector<DetectModel> models(K);
    std::vector<DetectCall> call(K);
    for (int k = 0; k < K; ++k) {
        models[k].role = roles[k]; models[k].stride = strides[k];
        call[k].n_steps = n_steps[k]; call[k].pending = pending[k];
    }
    return event_call_rows(models.data(), call.data(), pending_after, K);
}

// one timed models call (every model on all streams, as rows = streams); -1 when the pending rows give no common R
long long emul_timed_models(int n_streams, int K, const int *roles, const int *windows, const int *cooldowns, const double *cutoffs,
                            const int *strides, float *const *hist, long long *const *seen, int32_t *const *flag, const float *const *probs,
                            const long long *pitch, const int *n_steps, const int *pending, const int *pending_after, long long row_end,
                            int hop, mww_event *events, long long *positions, int capacity) {
    std::vector<DetectModel> models(K);
    DetectModelsArgs a;
    a.n_streams = n_streams; a.n_models = K; a.vad = -1; a.n_wake = 0; a.capacity = capacity;
    for (int k = 0; k < K; ++k) {
        DetectModel &M = models[k];
        M.role = roles[k];
        M.rule.window = windows[k]; M.rule.cutoff = cutoffs[k]; M.rule.cooldown_slices = cooldowns[k];
        M.stride = strides[k]; M.n_rows = n_streams;
        M.hist = hist[k]; M.seen = seen[k]; M.flag = flag[k];
        if (M.role == MWW_DETECT_VAD) a.vad = k;
        if (M.role == MWW_DETECT_WAKE) a.wake[a.n_wake++] = (int8_t)k;
        a.call[k].probs = probs[k]; a.call[k].pitch = pitch[k]; a.call[k].n_steps = n_steps[k]; a.call[k].pending = pending[k];
    }
    a.models = models.data();
    const long long R = event_call_rows(models.data(), a.call, pending_after, K);
    if (R < 0 || !detect_call_fits(models.data(), a.call, K)) return -1;
    ModelsSink sink{a, events, positions, capacity, 0, event_row0_end(row_end, hop, R), hop};
    const int lanes = (n_streams + 31) / 32 * 32;
    for (int s = 0; s < lanes; ++s) detect_models_stream(a, s, sink);
    return sink.count;
}

// the read-at kernel's units over rows x units (vec: 8-entry units, as the launcher picks them)
void emul_read_at(const int16_t *ring, int C, long long seen, const int32_t *ids, const long long *ends, int n, int n_streams, int n_samples,
                  int16_t *out, long long out_stride, int vec) {
    const int units = vec ? n_samples / 8 : n_samples;
    for (int r = 0; r < n; ++r) {
        const int id = ids[r];
        int16_t *dst = out + (long long)r * out_stride;
        for (int u = 0; u < units; ++u) {
            if (!vec) { dst[u] = history_at_one(ring, C, seen, id, n_streams, ends[r], n_samples, u); continue; }
            if (history_at_unit_in_ring(seen, C, id, n_streams, ends[r], n_samples, u, out_stride)) {
                const int16_t *src = ring + (long long)id * C + history_mod(ends[r] - n_samples + 8 * u, C);
                for (int q = 0; q < 8; ++q) dst[8 * u + q] = src[q];
            } else {
                for (int q = 0; q < 8; ++q) dst[8 * u + q] = history_at_one(ring, C, seen, id, n_streams, ends[r], n_samples, 8 * u + q);
            }
        }
    }
}

void emul_slots_at(long long count, int capacity, const mww_event *events, const long long *positions, int model, long long post, long long seen,
                   int C, int n_samples, int32_t *ids, long long *ends) {
    for (int i = 0; i < capacity; ++i) {
        const SlotAt s = verify_slot_at(i, count, capacity, events, positions, model, post, seen, C, n_samples);
        ids[i] = s.id;
        ends[i] = s.end;
    }
}

}  // extern "C"
