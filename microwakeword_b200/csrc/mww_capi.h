// mww_capi.h -- what the C-ABI translation units share: mww_capi.cu (the handle), mww_detector_capi.cu (the streaming
// detectors), mww_endpoint_capi.cu (the endpointer), mww_media_guard_capi.cu (the media guard), mww_verify_capi.cu (the
// verifier) and mww_playback_capi.cu (the playback guard).  Host code only.
#pragma once

#include <cuda_runtime.h>

#include <string>

#include "../../include/mww.h"

namespace mww {

// a refusal or failure: msg goes to the handle (mww_last_error(h)) or, for h == nullptr, to the calling thread's error of
// the last call without a handle (mww_last_error(NULL): a failed create, the detectors); returns code
int fail(mww_t *h, int code, const std::string &msg);
// MWW_ECUDA with "what: <CUDA error>"
int cuda_fail(mww_t *h, cudaError_t e, const char *what);

// every entry point runs with the handle's device current and puts the caller's device back on return (a process that
// holds engines on several GPUs, or torch's current device, is not disturbed)
struct DeviceGuard {
    int prev = -1; bool switched = false; cudaError_t err = cudaSuccess;
    explicit DeviceGuard(int device) {
        if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
        if (prev != device) { err = cudaSetDevice(device); switched = err == cudaSuccess && prev >= 0; }
    }
    ~DeviceGuard() { if (switched) cudaSetDevice(prev); }
};

// a handle's audio history as a kernel of another object reads it in stream order (the endpointer's command read): ring
// [n_streams][capacity] and samples_seen as of the calls issued so far.  ring is nullptr when the handle keeps no history;
// poisoned is set when a staged call failed half-way.
struct HistoryRing {
    const int16_t *ring; int capacity; long long seen; int n_streams, sm_count; bool poisoned;
};
HistoryRing history_ring(const mww_t *h);

// a detector's per-event-slot groups [capacity] (mww_drain_detector_groups' source) as the media guard's kernels read them;
// nullptr for a detector that is not grouped
const int32_t *detector_event_groups(const mww_detector_t *d);

// A verifier's scoring pass over the clips already in its clip buffer [slots][n_samples] (mww_verify_capi.cu):
// mww_reset(NULL) of its model handle, one mww_predict_clip over every slot and mww_positive_scores of the first n tracks into
// verifier_scores(v).  The verifier calls it after its history read; the playback guard after its reference read.
int16_t *verifier_clips(mww_verifier_t *v);
const float *verifier_scores(const mww_verifier_t *v);
int verifier_score_clips(mww_verifier_t *v, int n, cudaStream_t st, const std::string &call);

}  // namespace mww
