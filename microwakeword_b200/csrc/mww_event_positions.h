// mww_event_positions.h -- event positions on the audio history's axis (include/mww.h, "event positions"): where a timed
// detector's step ends, the history read that ends at given positions (mww_read_audio_history_at) and the verifier slots that
// end at their events (mww_verify_detections_at).  The kernels are in mww_event_positions.cu; the rule bodies they run are the
// detectors' own (mww_detector.h, mww_detector_models.h), the endpointer's ring-window read (mww_endpoint.h) and the
// verifier's slot rule (mww_verify.h).
//
// CUDA-free apart from MWW_HD, so that tests/emul_event_positions.cc runs the same functions on the CPU.
#pragma once

#include <stdint.h>

#include "../../include/mww.h"
#include "mww_common.h"
#include "mww_detector_models.h"
#include "mww_endpoint.h"
#include "mww_verify.h"

namespace mww {

// ---- where a step ends ----------------------------------------------------------------------------------------------------------
// Plain detector: a call of n steps on the clock (last_end, step_samples); step t ends at last_end - (n - 1 - t) step_samples.
// For an engine call last_end = endpoint_position(S, buffered, hop, g, stride, n, n - 1) and step_samples = hop * stride.
MWW_HD long long event_step_end(long long last_end, long long step_samples, int n, int t) {
    return last_end - (long long)(n - 1 - t) * step_samples;
}

// Models detector: a call that produced R feature rows, the newest ending at row_end = S - b (the frontend's b samples after
// it; endpoint_position's b).  Call-relative row e ends at row_end - hop (R - 1 - e), so row 0 ends at
//     row0_end = row_end - hop (R - 1),
// and WAKE step j of model k, which ends on row e_k(j) = (j + 1) s_k - p_k - 1 (detect_end_row), at row0_end + hop e_k(j).
// That is endpoint_position: with g_k = p_k + R - n_k s_k, the pending rows after the call,
//     row_end - hop (R - 1 - (j + 1) s_k + p_k + 1) = row_end - hop (g_k + (n_k - 1 - j) s_k).
MWW_HD long long event_row0_end(long long row_end, int hop, long long R) { return row_end - (long long)hop * (R - 1); }
MWW_HD long long event_model_step_end(long long row0_end, int hop, int j, int stride, int pending) {
    return row0_end + (long long)hop * detect_end_row(j, stride, pending);
}

// The rows a models call produced, from the step counts and each model's pending rows before and after it: R = n_k s_k - p_k
// + g_k for every non-OFF model, 0 <= p_k, g_k < s_k.  -1 when the models disagree or a count is out of range.  The step
// counts and p_k alone fix R only up to the strides (detect_call_fits); g_k fixes it.
inline long long event_call_rows(const DetectModel *models, const DetectCall *call, const int *pending_after, int n_models) {
    long long R = -1;
    for (int k = 0; k < n_models; ++k) {
        if (models[k].role == MWW_DETECT_OFF) continue;
        const long long s = models[k].stride, p = call[k].pending, g = pending_after[k], n = call[k].n_steps;
        if (n < 0 || p < 0 || p >= s || g < 0 || g >= s) return -1;
        const long long r = n * s - p + g;
        if (r < 0 || (R >= 0 && r != R)) return -1;
        R = r;
    }
    return R;
}

// ---- the read that ends at a position -------------------------------------------------------------------------------------------
// Row i of a read of n samples ending at `end`: entry k is axis position end - n + k of stream id, zero outside the ring
// [seen - C, seen) and for an id outside [0, n_streams) -- the endpointer's command read (endpoint_command_one).
MWW_HD int16_t history_at_one(const int16_t *ring, int C, long long seen, int id, int n_streams, long long end, int n, int k) {
    if (id < 0 || id >= n_streams) return 0;
    return endpoint_command_one(ring, C, seen, id, end - n + k);
}
// whether 8-entry unit u of that row is one aligned 16-byte load from the ring: its 8 positions in the ring, starting on a slot
// that is a multiple of 8 (history_read_vec_shape; the launcher adds n % 8, out_stride % 8 and the output's alignment)
MWW_HD bool history_at_unit_in_ring(long long seen, int C, int id, int n_streams, long long end, int n, int u, long long out_stride) {
    const long long t0 = end - n + 8 * u;
    return id >= 0 && id < n_streams && endpoint_in_ring(t0, seen, C) && endpoint_in_ring(t0 + 7, seen, C) &&
           history_read_vec_shape(history_mod(t0, C), n, out_stride);
}

// ---- verifier slots that end at their events ------------------------------------------------------------------------------------
// Slot i of a timed detector: verify_slot_id's stream, and the end of its clip e = min(P + post, S) for the slot's position P.
// The slot is scored only when the whole clip [e - n_samples, e) is still in the ring, e - n_samples >= S - C; otherwise, and
// for every slot verify_slot_id leaves at -1, id and end are -1.
struct SlotAt { int32_t id; long long end; };
MWW_HD SlotAt verify_slot_at(int i, long long count, int capacity, const mww_event *events, const long long *positions, int model,
                             long long post, long long seen, int C, int n_samples) {
    SlotAt s{verify_slot_id(i, count, capacity, events, model), -1};
    if (s.id < 0) return s;
    const long long p = positions[i] + post;
    const long long e = p < seen ? p : seen;
    if (e - n_samples < seen - C) { s.id = -1; return s; }
    s.end = e;
    return s;
}

}  // namespace mww
