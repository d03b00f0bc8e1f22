// mww_verify_capi.cu -- the extern "C" entry points of second-stage verification (include/mww.h).  Host code only: the two
// kernels are in mww_verify.{h,cu}.  A verifier is an object of its own, like a detector: it reads a source handle and a
// detector only through their public calls, runs its model on a handle of its own through the public clip path, and its
// messages go to mww_last_error(NULL).
#include <cmath>
#include <string>
#include <vector>

#include "mww_capi.h"
#include "mww_kernels.h"

using namespace mww;

struct mww_verifier {
    int device = 0, slots = 0, steps = 0;
    mww_verify_rule rule{};
    mww_t *h = nullptr;                 // the verifier's model on `slots` streams: scratch, fully reset by every call
    int16_t *d_audio = nullptr;         // [slots][n_samples] history read of the listed ids
    float *d_probs = nullptr;           // [slots][steps] the model's probabilities
    long long *d_offsets = nullptr;     // [slots] i * steps, the tracks mww_positive_scores reads
    int *d_lengths = nullptr;           // [slots] steps
    float *d_scores = nullptr;          // [slots] the positive scores of the first n tracks
    int32_t *d_ids = nullptr;           // [slots] a detector's slots as stream ids (mww_verify_detections)
    long long *d_ends = nullptr;        // [slots] the end of each slot's clip (mww_verify_detections_at)
};

namespace {

constexpr int kVerifyMaxSamples = 1 << 22;

#define VCU(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return cuda_fail(nullptr, e_, #call); } while (0)

int refuse(const std::string &msg) { return fail(nullptr, MWW_EINVAL, msg); }

// a failed call on another object: its code, with its message behind ours
int pass_on(int rc, const mww_t *h, const std::string &what) {
    const char *m = mww_last_error(h);
    return fail(nullptr, rc, what + ": " + (m ? m : "failed"));
}

void verifier_free(mww_verifier_t *v) {
    if (v->h) mww_destroy(v->h);
    cudaFree(v->d_audio); cudaFree(v->d_probs); cudaFree(v->d_offsets); cudaFree(v->d_lengths); cudaFree(v->d_scores); cudaFree(v->d_ids); cudaFree(v->d_ends);
    delete v;
}

// Every buffer of the verifier, and the clip scratch of its handle: one clip call on the zeroed staging sizes it, so that no
// verify call allocates.
int verifier_alloc(mww_verifier_t *v) {
    const size_t S = (size_t)v->slots, N = (size_t)v->rule.n_samples, M = (size_t)v->steps;
    VCU(cudaMalloc(&v->d_audio, S * N * sizeof(int16_t)));
    VCU(cudaMalloc(&v->d_probs, S * M * sizeof(float)));
    VCU(cudaMalloc(&v->d_offsets, S * sizeof(long long)));
    VCU(cudaMalloc(&v->d_lengths, S * sizeof(int)));
    VCU(cudaMalloc(&v->d_scores, S * sizeof(float)));
    VCU(cudaMalloc(&v->d_ids, S * sizeof(int32_t)));
    VCU(cudaMalloc(&v->d_ends, S * sizeof(long long)));
    std::vector<long long> offsets(S);
    for (size_t i = 0; i < S; ++i) offsets[i] = (long long)(i * M);
    const std::vector<int> lengths(S, v->steps);
    VCU(cudaMemcpy(v->d_offsets, offsets.data(), S * sizeof(long long), cudaMemcpyHostToDevice));
    VCU(cudaMemcpy(v->d_lengths, lengths.data(), S * sizeof(int), cudaMemcpyHostToDevice));
    VCU(cudaMemset(v->d_audio, 0, S * N * sizeof(int16_t)));
    int got = 0;
    if (int rc = mww_predict_clip(v->h, v->d_audio, v->rule.n_samples, v->rule.n_samples, v->d_probs, v->steps, &got, nullptr))
        return pass_on(rc, v->h, "mww_verifier_create");
    VCU(cudaDeviceSynchronize());
    return MWW_OK;
}

// The checks both verify calls share, before any device work: the verifier and src, src's audio history and device, the
// number of ids, and (probe: a read of nothing, which refuses a poisoned handle and launches nothing) src's health.
int check_source(const mww_verifier_t *v, mww_t *src, const std::string &call, int n, int *src_streams, cudaStream_t st) {
    if (!v || !src) return refuse(call + ": needs a verifier and a source handle");
    if (n < 0 || n > v->slots) return refuse(call + ": " + std::to_string(n) + " ids for a verifier of " + std::to_string(v->slots) + " slots");
    mww_info info;
    if (mww_get_info(src, &info) != MWW_OK) return refuse(call + ": cannot read the source handle");
    if (info.device != v->device) return refuse(call + ": the source handle is on another device than the verifier");
    int cap = 0;
    long long seen = 0;
    mww_get_audio_history(src, &cap, &seen);
    if (cap < v->rule.n_samples)
        return refuse(call + ": the source handle keeps " + (cap ? std::to_string(cap) + " samples of audio history" : std::string("no audio history")) +
                      "; the verifier reads " + std::to_string(v->rule.n_samples));
    if (mww_read_audio_history_device_ids(src, nullptr, 0, 0, nullptr, 0, st) != MWW_OK)
        return refuse(call + ": the source handle cannot be read: " + mww_last_error(src));
    *src_streams = info.n_streams;
    return MWW_OK;
}

// The pass over n ids in device memory: src's history of each (the last n_samples, or with d_ends the n_samples before
// d_ends[i]), their scores (verifier_score_clips), and the confirm kernel.  A constant number of launches for n >= 1.
int run(mww_verifier_t *v, mww_t *src, int src_streams, const int32_t *d_ids, const long long *d_ends, int n, float *d_scores,
        int32_t *d_confirmed, cudaStream_t st, const std::string &call) {
    const int N = v->rule.n_samples;
    const int rc = d_ends ? mww_read_audio_history_at(src, d_ids, d_ends, n, N, v->d_audio, N, st)
                          : mww_read_audio_history_device_ids(src, d_ids, n, N, v->d_audio, N, st);
    if (rc) return pass_on(rc, src, call + ": history read");
    if (int rc = verifier_score_clips(v, n, st, call)) return rc;
    VCU(launch_verify_confirm(d_ids, n, src_streams, v->d_scores, v->rule.cutoff, d_scores, d_confirmed, st));
    return MWW_OK;
}

// The checks both detector calls share, before any device work: the detector's buffers, its size against the slots, the
// source, the detector's device and the model index
int check_detections(mww_verifier_t *v, mww_t *src, mww_detector_t *det, int model, const std::string &call, const long long **d_count,
                     const mww_event **d_events, int *capacity, int *src_streams, cudaStream_t st) {
    if (!det) return refuse(call + ": detector is NULL");
    mww_detector_buffers(det, d_count, d_events, nullptr, capacity);
    if (v && *capacity > v->slots)
        return refuse(call + ": the detector keeps " + std::to_string(*capacity) + " events; the verifier has " + std::to_string(v->slots) + " slots");
    if (int rc = check_source(v, src, call, *capacity, src_streams, st)) return rc;
    cudaPointerAttributes attr;
    if (cudaPointerGetAttributes(&attr, *d_count) != cudaSuccess || attr.device != v->device) {
        cudaGetLastError();
        return refuse(call + ": the detector is on another device than the verifier");
    }
    mww_detector_layout layout;
    mww_get_detector_layout(det, &layout);
    if (model >= layout.n_models)
        return refuse(call + ": model " + std::to_string(model) + " of a detector of " + std::to_string(layout.n_models) + " model(s)");
    return MWW_OK;
}

}  // namespace

namespace mww {

int16_t *verifier_clips(mww_verifier_t *v) { return v->d_audio; }
const float *verifier_scores(const mww_verifier_t *v) { return v->d_scores; }

int verifier_score_clips(mww_verifier_t *v, int n, cudaStream_t st, const std::string &call) {
    const int N = v->rule.n_samples;
    if (int rc = mww_reset(v->h, nullptr, 0, st)) return pass_on(rc, v->h, call + ": verifier reset");
    int got = 0;
    if (int rc = mww_predict_clip(v->h, v->d_audio, N, N, v->d_probs, v->steps, &got, st)) return pass_on(rc, v->h, call + ": verifier clip");
    if (int rc = mww_positive_scores(v->d_probs, v->d_offsets, v->d_lengths, n, v->rule.window, v->rule.ignore_steps, v->d_scores, st))
        return fail(nullptr, rc, call + ": mww_positive_scores failed");
    return MWW_OK;
}

}  // namespace mww

extern "C" {

int mww_verifier_create(const void *model_blob, size_t n_bytes, int device, int slots, const mww_verify_rule *rule, mww_verifier_t **out) {
    const std::string call = "mww_verifier_create: ";
    if (!out) return refuse(call + "out is NULL");
    *out = nullptr;
    if (!rule) return refuse(call + "rule is NULL");
    if (slots < 1) return refuse(call + "slots must be at least 1");
    if (rule->n_samples < kWindow || rule->n_samples > kVerifyMaxSamples) return refuse(call + "n_samples must be in [480, 2^22]");
    if (rule->window < 1 || rule->window > kDetectorMaxWindow) return refuse(call + "window must be in [1, 32]");
    if (rule->ignore_steps < 0) return refuse(call + "ignore_steps must not be negative");
    if (!std::isfinite(rule->cutoff)) return refuse(call + "cutoff must be finite");
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0)
        return fail(nullptr, MWW_ECUDA, std::string("no CUDA device available (this library has no CPU fallback): ") + cudaGetErrorString(e));
    if (!model_blob || n_bytes == 0) return refuse(call + "a verifier needs a model (the blob is frontend-only)");
    mww_t *h = nullptr;
    if (int rc = mww_create(model_blob, n_bytes, device, slots, &h)) return rc;          // its message is mww_last_error(NULL) already
    mww_info info;
    mww_get_info(h, &info);
    const int frames = (rule->n_samples - kWindow) / kHop + 1;
    const int steps = frames / std::max(info.input_feature_slices, 1);
    if ((long long)steps < (long long)rule->ignore_steps + rule->window) {
        mww_destroy(h);
        return refuse(call + "the clip gives " + std::to_string(steps) + " probabilities, fewer than ignore_steps + window: every score would be NaN");
    }
    DeviceGuard guard(device);
    if (guard.err != cudaSuccess) { mww_destroy(h); return cuda_fail(nullptr, guard.err, "cudaSetDevice"); }
    mww_verifier_t *v = new mww_verifier;
    v->device = device; v->slots = slots; v->steps = steps; v->rule = *rule; v->rule.pad = 0; v->h = h;
    if (int rc = verifier_alloc(v)) { verifier_free(v); return rc; }
    *out = v;
    return MWW_OK;
}

int mww_verifier_destroy(mww_verifier_t *v) {
    if (!v) return MWW_OK;
    DeviceGuard guard(v->device);
    cudaDeviceSynchronize();
    verifier_free(v);
    return MWW_OK;
}

int mww_verifier_info(const mww_verifier_t *v, mww_verifier_desc *out) {
    if (!v || !out) return refuse("mww_verifier_info: needs a verifier and out");
    *out = mww_verifier_desc{};
    out->slots = v->slots; out->steps = v->steps; out->device = v->device; out->rule = v->rule;
    out->launches = mww_launch_count(v->h);
    return MWW_OK;
}

int mww_verify_streams(mww_verifier_t *v, mww_t *src, const int32_t *d_ids, int n, float *d_scores, int32_t *d_confirmed, void *cu_stream) {
    const std::string call = "mww_verify_streams";
    cudaStream_t st = static_cast<cudaStream_t>(cu_stream);
    int src_streams = 0;
    if (int rc = check_source(v, src, call, n, &src_streams, st)) return rc;
    if (n > 0 && !d_ids) return refuse(call + ": d_ids is NULL");
    if (n == 0) return MWW_OK;
    DeviceGuard guard(v->device);
    if (guard.err != cudaSuccess) return cuda_fail(nullptr, guard.err, "cudaSetDevice");
    return run(v, src, src_streams, d_ids, nullptr, n, d_scores, d_confirmed, st, call);
}

int mww_verify_detections(mww_verifier_t *v, mww_t *src, mww_detector_t *det, int model, float *d_scores, int32_t *d_confirmed,
                          void *cu_stream) {
    const std::string call = "mww_verify_detections";
    const long long *d_count = nullptr;
    const mww_event *d_events = nullptr;
    int capacity = 0, src_streams = 0;
    cudaStream_t st = static_cast<cudaStream_t>(cu_stream);
    if (int rc = check_detections(v, src, det, model, call, &d_count, &d_events, &capacity, &src_streams, st)) return rc;
    DeviceGuard guard(v->device);
    if (guard.err != cudaSuccess) return cuda_fail(nullptr, guard.err, "cudaSetDevice");
    VCU(launch_verify_slots(d_count, d_events, capacity, model, v->d_ids, st));
    return run(v, src, src_streams, v->d_ids, nullptr, capacity, d_scores, d_confirmed, st, call);
}

int mww_verify_detections_at(mww_verifier_t *v, mww_t *src, mww_detector_t *det, int model, long long post, float *d_scores, int32_t *d_confirmed,
                             void *cu_stream) {
    const std::string call = "mww_verify_detections_at";
    if (post < 0 || post > kVerifyMaxSamples) return refuse(call + ": post must be in [0, 2^22]");
    const int64_t *d_positions = nullptr;
    if (det && mww_get_detector_positions(det, &d_positions) != MWW_OK)
        return refuse(call + ": the detector is not timed (mww_time_detector_events): its events carry no positions");
    const long long *d_count = nullptr;
    const mww_event *d_events = nullptr;
    int capacity = 0, src_streams = 0;
    cudaStream_t st = static_cast<cudaStream_t>(cu_stream);
    if (int rc = check_detections(v, src, det, model, call, &d_count, &d_events, &capacity, &src_streams, st)) return rc;
    int C = 0;
    long long S = 0;
    mww_get_audio_history(src, &C, &S);
    DeviceGuard guard(v->device);
    if (guard.err != cudaSuccess) return cuda_fail(nullptr, guard.err, "cudaSetDevice");
    VCU(launch_verify_slots_at(d_count, d_events, reinterpret_cast<const long long *>(d_positions), capacity, model, post, S, C, v->rule.n_samples,
                               v->d_ids, v->d_ends, st));
    return run(v, src, src_streams, v->d_ids, v->d_ends, capacity, d_scores, d_confirmed, st, call);
}

}  // extern "C"
