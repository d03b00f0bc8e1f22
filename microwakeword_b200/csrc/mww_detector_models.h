// mww_detector_models.h -- the multi-model streaming detector (mww_multi_detector_create, include/mww.h): one detector over
// the K models of a handle, a rule per model (WAKE, VAD or OFF), the WAKE models' detections gated by the VAD's.  The
// per-stream body detector_models_update_kernel runs for every stream (mww_detector_models.cu); CUDA-free apart from MWW_HD,
// so that tests/emul_detector_models.cc runs the same functions on the CPU.
//
// Definition (include/mww.h states it in full).  Model k of stride s_k that held p_k pending rows before a call and ran
// n_k steps in it ends its step j at call-relative feature row e_k(j) = (j + 1) s_k - p_k - 1.  A stream's steps are
// processed in order of e, a VAD step before a WAKE step that ends on the same row.  A VAD step sets the stream's `active`
// flag to (seen >= window && (double)avg > cutoff); a WAKE step is mww_detector.h's rule with one more condition on firing:
// the stream's VAD row is active (true when no model is the VAD; false for a stream the VAD does not score).  WAKE models
// do not depend on each other, so only the VAD's steps order the work: the thread walks the VAD's steps and, before each,
// the WAKE steps that end below it.
#pragma once

#include <stdint.h>

#include <type_traits>

#include "mww_detector.h"

namespace mww {

constexpr int kDetectMaxModels = 64;         // mww_create_multi's limit

// one model of a models detector, fixed at create: its rule and its rows' state, struct-of-arrays over the members of its
// stream set in list order (hist [window - 1][n_rows], so a thread per stream reads and writes it coalesced where row = stream)
struct DetectModel {
    int role = MWW_DETECT_OFF;
    DetectorRule rule;                       // cutoff and window for every role, cooldown_slices for WAKE
    int stride = 1, n_rows = 0;
    const int32_t *inv = nullptr;            // [n_streams]: row of each stream, -1 for a non-member; nullptr: row = stream
    float *hist = nullptr;
    long long *seen = nullptr;
    int32_t *flag = nullptr;                 // cooldown (WAKE) or active (VAD)
};

// model k's part of one update call
struct DetectCall {
    const float *probs = nullptr;            // [n_rows][pitch], the first n_steps columns read
    long long pitch = 0;
    int n_steps = 0, pending = 0;            // steps run in the call, pending rows before it
};

// a model's descriptor in per-row mode (mww_set_multi_detector_cutoffs): the same, and the cutoff of each of its rows
struct DetectModelRows : DetectModel {
    const double *row_cutoff = nullptr;      // [n_rows], list order
};

// The cutoff row `row` of model m compares against (row -1: a non-member, never compared).  Uniform mode reads the rule's
// where the comparison is; per-row mode loads the row's where it loads the row's state (for a WAKE row, once per VAD step).
struct RuleCutoff {
    const DetectModel *m = nullptr;
    MWW_HD double get() const { return m->rule.cutoff; }
};
MWW_HD RuleCutoff detect_cutoff(const DetectModel &m, int) { return RuleCutoff{&m}; }
MWW_HD CutoffValue detect_cutoff(const DetectModelRows &m, int row) { return CutoffValue{row >= 0 ? m.row_cutoff[row] : 0.0}; }

// what the update and reset kernels get: descriptors (device memory), the event buffer, its counter and the fired-id list
// shared with the plain detector, and the call -- pointers, pitches and step timing travel in the parameters, not by copy.
// M: DetectModel, or DetectModelRows in per-row mode.
template <typename M>
struct DetectModelsArgsT {
    int n_streams = 0, n_models = 0, vad = -1, n_wake = 0, capacity = 0;
    const M *models = nullptr;
    unsigned long long *count = nullptr;
    mww_event *events = nullptr;
    int32_t *fired = nullptr;
    int8_t wake[kDetectMaxModels] = {};      // the WAKE models' indices
    DetectCall call[kDetectMaxModels];
};
using DetectModelsArgs = DetectModelsArgsT<DetectModel>;

// the same arguments over per-row descriptors
inline DetectModelsArgsT<DetectModelRows> detect_args_rows(const DetectModelsArgs &a, const DetectModelRows *models) {
    DetectModelsArgsT<DetectModelRows> r;
    r.n_streams = a.n_streams; r.n_models = a.n_models; r.vad = a.vad; r.n_wake = a.n_wake; r.capacity = a.capacity;
    r.models = models; r.count = a.count; r.events = a.events; r.fired = a.fired;
    for (int k = 0; k < kDetectMaxModels; ++k) { r.wake[k] = a.wake[k]; r.call[k] = a.call[k]; }
    return r;
}

// one row's history, entry j at h[j * stride]
struct DetectHistory {
    float *h; long long stride;
    MWW_HD float get(int j) const { return h[j * stride]; }
    MWW_HD void set(int j, float v) const { h[j * stride] = v; }
};

// the mean of the row's last window - 1 probabilities and p, summed oldest first with one division (detector_window_mean's
// arithmetic), streamed as detector_step streams it: entry j is read, summed and written back to j - 1; p becomes the newest
MWW_HD float detect_push(const DetectHistory &hist, int w, float p) {
    float s = p;
    if (w > 1) {
        s = hist.get(0);
        for (int j = 1; j < w - 1; ++j) {
            const float v = hist.get(j);
            s = det_add(s, v);
            hist.set(j - 1, v);
        }
        s = det_add(s, p);
        hist.set(w - 2, p);
    }
    return det_div(s, (float)w);
}

// end row of step j of a model with stride s and p pending rows before the call
MWW_HD long long detect_end_row(int j, int s, int p) { return (long long)(j + 1) * s - p - 1; }

// how many of the call's n steps (stride s, p pending before) end below `row` (row >= 0)
MWW_HD int detect_steps_below(long long row, int s, int p, int n) {
    const long long c = (row + p) / s;
    return c > n ? n : (int)c;
}

// model m's row of `stream`, -1 for a non-member or a stream past the handle's (the idle lanes of the last warp)
MWW_HD int detect_row(const DetectModel &m, int stream, int n_streams) {
    if (stream >= n_streams) return -1;
    return m.inv ? m.inv[stream] : stream;
}

// Whether one R >= 0 (the feature rows the call produced) gives every non-OFF model n_k = (p_k + R) div s_k with
// 0 <= p_k < s_k: the update's consistency check, on the host before any launch.
inline bool detect_call_fits(const DetectModel *models, const DetectCall *call, int n_models) {
    long long lo = 0, hi = -1;
    bool any = false;
    for (int k = 0; k < n_models; ++k) {
        if (models[k].role == MWW_DETECT_OFF) continue;
        const long long s = models[k].stride, p = call[k].pending, n = call[k].n_steps;
        if (n < 0 || p < 0 || p >= s) return false;
        const long long a = n * s - p, b = (n + 1) * s - p - 1;      // (p + R) div s == n  <=>  a <= R <= b
        if (!any || a > lo) lo = a;
        if (!any || b < hi) hi = b;
        any = true;
    }
    if (lo < 0) lo = 0;
    return any && lo <= hi;
}

// emit(fire, k, stream, step, score, j), j the step's index in the call, where Emit takes it (the timed kernel places the
// event with it); emit(fire, k, stream, step, score) otherwise
template <typename Emit>
MWW_HD void detect_emit(Emit &emit, bool fire, int k, int stream, long long step, float score, int j) {
    if constexpr (std::is_invocable_v<Emit &, bool, int, int, long long, float, int>) emit(fire, k, stream, step, score, j);
    else emit(fire, k, stream, step, score);
}

// One call for one stream.  emit(fire, k, stream, step, score[, j]) is called for every WAKE step of every WAKE model in the
// same order on every stream, member or not (fire false for a non-member), so that the kernel's warps can ballot on it.
template <typename M, typename Emit>
MWW_HD void detect_models_stream(const DetectModelsArgsT<M> &a, int stream, Emit &emit) {
    const M *V = a.vad >= 0 ? &a.models[a.vad] : nullptr;
    int n_v = 0, vrow = -1, s_v = 1, p_v = 0;
    long long vseen = 0;
    decltype(detect_cutoff(*V, 0)) vcut;
    bool active = V == nullptr;                                  // no VAD: the gate is open
    if (V) {
        n_v = a.call[a.vad].n_steps; s_v = V->stride; p_v = a.call[a.vad].pending;
        vrow = detect_row(*V, stream, a.n_streams);
        if (vrow >= 0) { vseen = V->seen[vrow]; active = V->flag[vrow] != 0; }
        vcut = detect_cutoff(*V, vrow);
    }
    for (int i = 0; i <= n_v; ++i) {
        // the WAKE steps ending in [end of VAD step i - 1, end of VAD step i): they see the flag VAD step i - 1 left
        for (int w = 0; w < a.n_wake; ++w) {
            const int k = a.wake[w];
            const DetectCall &c = a.call[k];
            const M &W = a.models[k];
            const int j0 = i == 0 ? 0 : detect_steps_below(detect_end_row(i - 1, s_v, p_v), W.stride, c.pending, c.n_steps);
            const int j1 = i == n_v ? c.n_steps : detect_steps_below(detect_end_row(i, s_v, p_v), W.stride, c.pending, c.n_steps);
            if (j0 >= j1) continue;
            const int row = detect_row(W, stream, a.n_streams);
            long long seen = 0;
            int cooldown = 0;
            if (row >= 0) { seen = W.seen[row]; cooldown = W.flag[row]; }
            const auto cutoff = detect_cutoff(W, row);
            const DetectHistory hist{W.hist + (row >= 0 ? row : 0), W.n_rows};
            for (int j = j0; j < j1; ++j) {
                bool fire = false;
                float avg = 0.f;
                if (row >= 0) {
                    avg = detect_push(hist, W.rule.window, c.probs[row * c.pitch + j]);
                    if (seen + 1 >= W.rule.window) {                // warming up: no average, no tick
                        if (active) fire = detector_tick_from(W.rule, cutoff, avg, cooldown);
                        else cooldown = cooldown > 0 ? cooldown - 1 : 0;
                    }
                    ++seen;
                }
                detect_emit(emit, fire, k, stream, seen - 1, avg, j);
            }
            if (row >= 0) { W.seen[row] = seen; W.flag[row] = cooldown; }
        }
        if (i < n_v && vrow >= 0) {
            const DetectCall &c = a.call[a.vad];
            const float avg = detect_push(DetectHistory{V->hist + vrow, V->n_rows}, V->rule.window, c.probs[vrow * c.pitch + i]);
            ++vseen;
            active = vseen >= V->rule.window && (double)avg > vcut.get();
        }
    }
    if (vrow >= 0) { V->seen[vrow] = vseen; V->flag[vrow] = active ? 1 : 0; }
}

// fresh state of every non-OFF row of `stream` (a stream out of range is ignored): zero history, seen 0, cooldown_slices
// (WAKE) or inactive (VAD)
MWW_HD void detect_models_reset_stream(const DetectModelsArgs &a, long long stream) {
    if (stream < 0 || stream >= a.n_streams) return;
    for (int k = 0; k < a.n_models; ++k) {
        const DetectModel &M = a.models[k];
        if (M.role == MWW_DETECT_OFF) continue;
        const int row = detect_row(M, (int)stream, a.n_streams);
        if (row < 0) continue;
        for (int j = 0; j < M.rule.window - 1; ++j) M.hist[(long long)j * M.n_rows + row] = 0.f;
        M.seen[row] = 0;
        M.flag[row] = M.role == MWW_DETECT_WAKE ? M.rule.cooldown_slices : 0;
    }
}

}  // namespace mww
