// mww_verify.h -- the per-element bodies of the two kernels of second-stage verification (mww_verify.cu; rule in
// include/mww.h, "second-stage verification"): which stream a detector's event slot names, and how a verifier score becomes
// a confirmed stream id.  The frontend, the network and the score rule are not here: a verify call runs the existing
// history read, clip and positive-score paths through their public calls (mww_verify_capi.cu).
//
// CUDA-free apart from MWW_HD, so that tests/emul_verify.cc runs the same functions on the CPU.
#pragma once

#include <stdint.h>

#include "../../include/mww.h"
#include "mww_common.h"

namespace mww {

// Slot i of a detector's event buffer [capacity], `count` events having fired since its last drain: the stream of event i
// when the slot is used (i < min(count, capacity)) and the event belongs to `model` (model < 0: any model), else -1.
MWW_HD int32_t verify_slot_id(int i, long long count, int capacity, const mww_event *events, int model) {
    const long long used = count < (long long)capacity ? count : (long long)capacity;
    if ((long long)i >= used) return -1;
    const mww_event e = events[i];
    return (model < 0 || e.reserved == model) ? e.stream : -1;
}

// Index i of a verify call: the id it names and the score of the verifier's track for that index.  An id outside
// [0, n_streams) has no score (NaN) and confirms nothing; any other keeps its score and is confirmed when (double)score >
// cutoff, which NaN never is.
struct VerifyOut { float score; int32_t confirmed; };
MWW_HD VerifyOut verify_confirm(int32_t id, int n_streams, float score, double cutoff) {
    VerifyOut o;
    const bool listed = id >= 0 && id < n_streams;
    o.score = listed ? score : __builtin_nanf("");
    o.confirmed = listed && (double)score > cutoff ? id : -1;
    return o;
}

}  // namespace mww
