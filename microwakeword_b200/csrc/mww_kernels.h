// mww_kernels.h -- launcher prototypes shared by the C-ABI layer (mww_capi.cu, mww_detector_capi.cu) and the kernel files.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "mww_tables.h"

namespace mww {

// Dynamic shared memory above 48 KB is opt-in per kernel AND per device (cudaFuncSetAttribute applies to the current
// device only): a process that drives several GPUs must opt in on each of them.  `done` is the launcher's static flag set.
inline bool first_launch_on_this_device(bool (&done)[64]) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return true;
    if (done[dev]) return false;
    done[dev] = true;
    return true;
}

// Every launcher that reads caller audio is instantiated for T = int16_t (PCM) and T = float (float32 in [-1, 1], converted
// on load with pcm16_from_f32) in libmww_b200.so, and for T = Ulaw8 and Alaw8 (G.711 bytes, decoded on load) in
// libmww_g711.so (mww_frontend_g711.cu); the window carry is int16 whatever T is, so calls of all four types can follow
// each other.
template <typename T>
cudaError_t launch_k1(const FrontendParams &P, const int16_t *carry, int used, const T *audio,
                      long long audio_stride, int n_samples, int n_streams, int n_frames, uint32_t *vout, int sm_count,
                      cudaStream_t st);
// long calls with enough streams for one CTA per stream: K1 + the temporal chain in one launch, features written directly
// (no V scratch).  frontend_clip_fuses() is the predicate the C-ABI layer sizes its scratch with.
bool frontend_clip_fuses(int n_streams, int n_frames, int sm_count);
template <typename T>
cudaError_t launch_frontend_clip_fused(const FrontendParams &P, const int16_t *carry, int used, const T *audio, long long audio_stride,
                                       int n_samples, int n_streams, int n_frames, uint32_t *estimate, uint16_t *feat, long long feat_stream_stride,
                                       cudaStream_t st);
// the same features from k1_clip_kernel (mww_frontend_clip.cu, companion library libmww_frontend_clip.so): half-warp barriers
// between the per-frame phases.  The C-ABI layer runs it for every fused clip call except under MWW_K1_OCC=3, which selects
// launch_frontend_clip_fused's 3-CTA instantiation.
template <typename T>
cudaError_t launch_frontend_clip(const FrontendParams &P, const int16_t *carry, int used, const T *audio, long long audio_stride,
                                 int n_samples, int n_streams, int n_frames, uint32_t *estimate, uint16_t *feat, long long feat_stream_stride,
                                 cudaStream_t st);
// any even hop <= 480 samples (window_step != 10 ms): K1 + temporal chain, one CTA per stream, features written directly
template <typename T>
cudaError_t launch_frontend_hop(const FrontendParams &P, const int16_t *carry, int used, const T *audio, long long audio_stride,
                                int n_samples, int n_streams, int n_frames, int hop, uint32_t *estimate, uint16_t *feat,
                                long long feat_stream_stride, cudaStream_t st);
// short calls (<= 8 frames per stream, <= 2 hops left over): K1 + K2 + carry update in one launch
bool frontend_fusable(int used, int n_samples, int n_frames);
template <typename T>
cudaError_t launch_frontend_fused(const FrontendParams &P, int16_t *carry, int used, const T *audio,
                                  long long audio_stride, int n_samples, int n_streams, int n_frames, uint32_t *estimate, uint16_t *feat,
                                  long long feat_stream_stride, cudaStream_t st);
cudaError_t launch_k2(const FrontendParams &P, const uint32_t *vin, int n_streams, int n_frames, uint32_t *estimate,
                      uint16_t *feat, long long feat_stream_stride, cudaStream_t st);
template <typename T>
cudaError_t launch_carry_update(int16_t *carry, int used, const T *audio, long long audio_stride, int n_samples,
                                int n_streams, int consumed, int new_used, cudaStream_t st);

}  // namespace mww

#include "mww_nn_dev.cuh"
namespace mww {
cudaError_t launch_nn_f32(const NnWeightsF32 &W, float *state, float *pend, int n_pend, const void *rows,
                          long long rows_stream_stride_bytes, int n_rows, int rows_are_f32, float *probs,
                          long long probs_stream_stride, float *logits, int n_streams, cudaStream_t st);
}  // namespace mww

#include "mww_nn_i8_dev.cuh"
namespace mww {
cudaError_t launch_nn_i8(const NnWeightsI8 &W, int8_t *state, int8_t *pend, int n_pend, const void *rows,
                         long long rows_stream_stride_bytes, int n_rows, int row_type, float *probs,
                         long long probs_stream_stride, int n_streams, cudaStream_t st);
// zero-point fill of streams 0 .. n (ids == nullptr) or of the n listed streams
cudaError_t launch_fill_state_i8(const NnWeightsI8 &W, int8_t *state, int8_t *pend, const int32_t *ids, int n, int n_streams, cudaStream_t st);
}  // namespace mww

#include "mww_nn_live.cuh"
namespace mww {
// live-step path (one model step for many streams per launch; mww_nn_live.cuh).  `heads` = current rotation of the rings;
// the caller advances every head by one (mod its ring length) after the launch.
cudaError_t launch_nn_f32_live(const NnWeightsF32 &W, float *state, float *pend, int n_pend, const void *rows,
                               long long rows_stream_stride_bytes, int rows_are_f32, float *probs, long long probs_stride,
                               int n_streams, const LiveHeads &heads, int sm_count, int variant, cudaStream_t st);
// rotate every ring of every stream back to the canonical oldest-first layout (no-op rings with head 0 are skipped)
cudaError_t launch_nn_live_canonicalise(float *state, int n_streams, const LiveHeads &heads, cudaStream_t st);
// int8 live-step path (mww_nn_i8_live.cuh); rows must be 16-byte aligned with a 16-byte-multiple stream stride
cudaError_t launch_nn_i8_live(const NnWeightsI8 &W, int8_t *state, int8_t *pend, int n_pend, const void *rows,
                              long long rows_stream_stride_bytes, int row_type, float *probs, long long probs_stride, int n_streams,
                              const LiveHeads &heads, int sm_count, cudaStream_t st);
cudaError_t launch_nn_i8_live_canonicalise(int8_t *state, int n_streams, const LiveHeads &heads, cudaStream_t st);
}  // namespace mww

#include "mww_nn_generic.cuh"
namespace mww {
// run-time-geometry MixedNet (any architecture other than the compiled-in okay_nabu one; mww_nn_generic.cuh)
cudaError_t launch_nn_generic_f32(const GenArch &A, const GenWeightsF32 &W, float *state, float *pend, int n_pend, const void *rows,
                                  long long rows_stream_stride_bytes, int n_rows, int row_type, float *probs, long long probs_stream_stride,
                                  int n_streams, cudaStream_t st);
cudaError_t launch_nn_generic_i8(const GenArch &A, const GenWeightsI8 &W, int8_t *state, int8_t *pend, int n_pend, const void *rows,
                                 long long rows_stream_stride_bytes, int n_rows, int row_type, float *probs, long long probs_stream_stride,
                                 int n_streams, cudaStream_t st);
cudaError_t launch_gen_fill_state_i8(const GenArch &A, const GenWeightsI8 &W, int8_t *state, int8_t *pend, int n, const int32_t *ids, int n_streams,
                                     cudaStream_t st);
// fp32 graph with int8-weight (hybrid) ops, any architecture including okay_nabu's; fp32 state layout
cudaError_t launch_nn_generic_hybrid(const GenArch &A, const GenWeightsF32 &W, const GenHybrid &H, float *state, float *pend, int n_pend,
                                     const void *rows, long long rows_stream_stride_bytes, int n_rows, int row_type, float *probs,
                                     long long probs_stream_stride, int n_streams, cudaStream_t st);

// per-model stream sets (mww_streams.cu, index math in mww_streams.h)
// rows [n_rows][40] of the m members ids[a, a + m) of the tile whose rows start at stream `first` -> compact out [m][n_rows][40]
cudaError_t launch_gather_rows(const uint16_t *feat, const int32_t *ids, int a, int first, int m, int n_rows, uint16_t *out, int sm_count,
                               cudaStream_t st);
// new row j of dst [n_new][bytes_per_row] = old row old_index[j] of src; rows with old_index -1 are not written
cudaError_t launch_remap_rows(void *dst, const void *src, size_t bytes_per_row, const int32_t *old_index, int n_new, int sm_count,
                              cudaStream_t st);
// out[i] = compact index of global stream id ids[i] from the inverse map inv[n_streams], -1 for a non-member or an id out of range
cudaError_t launch_compact_ids(int32_t *out, const int32_t *ids, int n, const int32_t *inv, int n_streams, int sm_count, cudaStream_t st);
}  // namespace mww

#include "mww_resample.h"
namespace mww {
// input-rate resampler (mww_resample.cu, definition and index math in mww_resample.h): a tile's input samples -> its 16 kHz
// int16 samples out [n_streams][out_stride], history moved on.  T = int16_t or float (pcm16_from_f32 on load), or
// Ulaw8 / Alaw8 (decoded on load; instantiated in libmww_g711.so).
template <typename T>
cudaError_t launch_resample(const ResampleArgs &a, const T *audio, int16_t *out, int sm_count, cudaStream_t st);
// the same for the a.n_streams members ids[0, n) (device memory, sorted global ids) of one rate in the tile that starts at
// stream `first`: audio and out rows ids[i] - first, history rows ids[i] of a.hist (not offset).  A plan without taps
// (a.T == 0, 16 kHz) copies pcm16 of the input.
template <typename T>
cudaError_t launch_resample_members(const ResampleArgs &a, const int32_t *ids, int first, const T *audio, int16_t *out, int sm_count,
                                    cudaStream_t st);
// the same with a sample format per stream (MixedRows, mww_resample.h): audio is bytes, a.audio_stride counts bytes, and
// member ids[i] reads its row in format formats[ids[i]] (device memory [n_streams]); base and stride multiples of 4.
// Instantiated in libmww_resample_mixed.so.
cudaError_t launch_resample_mixed(const ResampleArgs &a, const int32_t *ids, int first, const uint8_t *formats, const Mixed8 *audio,
                                  int16_t *out, int sm_count, cudaStream_t st);
}  // namespace mww

#include "mww_records.h"
namespace mww {
// stream records (mww_records.cu, layout and index math in mww_records.h): the parts of job J of the n streams ids[0, n)
// between the handle (base[p]: part p of stream / compact index 0) and records [n][record_bytes].  inv: the model's
// compact index of each global stream id, nullptr for the frontend parts.  Unpack also writes fresh[0, n) when given:
// the compact index of each listed member the records hold no state for, else -1 (a job with zero_fresh zeroes them itself).
cudaError_t launch_pack_streams(const RecordJob &J, void *records, long long record_bytes, const int32_t *ids, int n, const void *const *base,
                                const int32_t *inv, int sm_count, cudaStream_t st);
cudaError_t launch_unpack_streams(const RecordJob &J, const void *records, long long record_bytes, const int32_t *ids, int n, void *const *base,
                                  const int32_t *inv, int32_t *fresh, int sm_count, cudaStream_t st);
}  // namespace mww

#include "mww_detector.h"
namespace mww {
// streaming detector (mww_detector.cu, rule and kernel forms in mww_detector.h): every row consumes the first n_steps
// columns of probs [n_rows][pitch]; thread per row below kDetectorWarpMinSteps steps, warp per row from there on
cudaError_t launch_detector_update(const DetectorArgs &a, const float *probs, int n_steps, long long pitch, cudaStream_t st);
// fresh state for the n listed rows (device memory; indices out of range ignored) or, rows == nullptr, for rows [0, n)
cudaError_t launch_detector_reset(const DetectorArgs &a, const int32_t *rows, int n, cudaStream_t st);
}  // namespace mww

#include "mww_detector_models.h"
namespace mww {
// multi-model detector (mww_detector_models.cu, rule and per-stream body in mww_detector_models.h): one call of every model,
// a thread per stream of the handle
cudaError_t launch_detector_models_update(const DetectModelsArgs &a, cudaStream_t st);
// fresh state of every model's row of the n listed GLOBAL stream ids (device memory; out of range ignored) or, ids ==
// nullptr, of streams [0, n)
cudaError_t launch_detector_models_reset(const DetectModelsArgs &a, const int32_t *ids, int n, cudaStream_t st);

// both detectors in per-row mode (mww_detector_cutoffs.cu): launch_detector_update with row r compared against
// row_cutoff[r] (device memory, [n_rows]), and launch_detector_models_update over descriptors that carry their rows' cutoffs
cudaError_t launch_detector_update_cutoffs(const DetectorArgs &a, const double *row_cutoff, const float *probs, int n_steps, long long pitch,
                                           cudaStream_t st);
cudaError_t launch_detector_models_update_cutoffs(const DetectModelsArgsT<DetectModelRows> &a, cudaStream_t st);
}  // namespace mww

#include "mww_detector_records.h"
namespace mww {
// detector records (mww_detector_records.cu, layout and per-word bodies in mww_detector_records.h; companion library
// libmww_detector_records.so): every used model's slot of the n records [n][J.words] of ids[0, n) (device memory, in range),
// one launch each way
cudaError_t launch_pack_detector_rows(const DetRecJob &J, void *records, const int32_t *ids, int n, cudaStream_t st);
cudaError_t launch_unpack_detector_rows(const DetRecJob &J, const void *records, const int32_t *ids, int n, cudaStream_t st);
}  // namespace mww

namespace mww {
// audio history (mww_history.cu, ring layout and index math in mww_history.h; companion library libmww_history.so)
// the last min(n16, C) of a call's n16 16 kHz samples of streams [0, n_streams) of `audio` (pcm16 of T on load) -> their
// slots of ring [n_streams][C], `seen` samples having come before the call
template <typename T>
cudaError_t launch_history_append(int16_t *ring, int C, long long seen, const T *audio, long long audio_stride, int n16, int n_streams,
                                  int sm_count, cudaStream_t st);
// out [n][out_stride]: row i = the last n_samples (<= C) of ring row ids[i] (device memory), zeros for an id outside [0, n_streams)
cudaError_t launch_history_read(const int16_t *ring, int C, long long seen, const int32_t *ids, int n, int n_streams, int n_samples, int16_t *out,
                                long long out_stride, int sm_count, cudaStream_t st);
}  // namespace mww

#include "mww_verify.h"
namespace mww {
// second-stage verification (mww_verify.cu, per-element bodies in mww_verify.h; companion library libmww_verify.so)
// ids [capacity]: the stream of each of a detector's event slots that holds an event of `model` (< 0: any), -1 elsewhere;
// *count is read on the device
cudaError_t launch_verify_slots(const long long *count, const mww_event *events, int capacity, int model, int32_t *ids, cudaStream_t st);
// out_scores / out_confirmed [n] (either may be nullptr) from the ids [n] and the verifier's scores [n]
cudaError_t launch_verify_confirm(const int32_t *ids, int n, int n_streams, const float *scores, double cutoff, float *out_scores,
                                  int32_t *out_confirmed, cudaStream_t st);
}  // namespace mww

#include "mww_endpoint.h"
namespace mww {
// endpointing (mww_endpoint.cu, rule and per-row bodies in mww_endpoint.h; companion library libmww_endpoint.so), one launch
// each.  update: n steps of every row, step j at position pos0 + j * a.step_samples
cudaError_t launch_endpoint_update(const EndpointArgs &a, const float *probs, long long pitch, int n, long long pos0, cudaStream_t st);
// arm the n listed global ids (device memory; ids outside the set ignored) with the replay R
cudaError_t launch_endpoint_arm(const EndpointArgs &a, const EndpointReplay &R, const int32_t *ids, int n, cudaStream_t st);
// disarm (reset 0) or reset (reset 1) the n listed global ids, or, ids == nullptr, rows [0, n)
cudaError_t launch_endpoint_clear(const EndpointArgs &a, const int32_t *ids, int n, int reset, cudaStream_t st);
// out [capacity][out_stride] and lengths [capacity]: the command of each used event slot from ring [n_streams][C], `seen`
// samples appended; *count is read on the device
cudaError_t launch_endpoint_read(const int16_t *ring, int C, long long seen, const unsigned long long *count, const mww_endpoint_event *events,
                                 int capacity, long long pre, long long post, int max_samples, int16_t *out, long long out_stride,
                                 int32_t *lengths, int sm_count, cudaStream_t st);
}  // namespace mww

#include "mww_serving_records.h"
namespace mww {
// moving a stream's serving state (mww_serving_records.cu, index math in mww_history.h, record layout and per-row bodies in
// mww_serving_records.h; companion library libmww_serving_records.so), one launch each.
// ring rows ids[i] (device memory, in range, distinct) of ring [n_streams][C] <- zeros followed by the n_samples of row i of
// in [n][in_stride], `seen` samples appended
cudaError_t launch_history_write(int16_t *ring, int C, long long seen, const int32_t *ids, int n, int n_samples, const int16_t *in,
                                 long long in_stride, int sm_count, cudaStream_t st);
// the records [n][J.L.record_bytes] of the n listed global ids (device memory, in range) out of and into the endpointer J
cudaError_t launch_pack_endpointer_rows(const EpRecJob &J, void *records, const int32_t *ids, int n, cudaStream_t st);
cudaError_t launch_unpack_endpointer_rows(const EpRecJob &J, const void *records, const int32_t *ids, int n, cudaStream_t st);

// the positioned endpointer (mww_endpoint_at.cu, bodies in mww_endpoint.h and mww_serving_records.h; companion library
// libmww_endpoint_at.so): the forms above that also keep each row's mute word mute [n_rows], one launch each, and arm_at, two
// launches (the reduction of each row's latest position, then the arm) of the n listed global ids and positions (device memory)
cudaError_t launch_endpoint_update_muted(const EndpointArgs &a, int32_t *mute, const float *probs, long long pitch, int n, long long pos0,
                                         cudaStream_t st);
cudaError_t launch_endpoint_arm_muted(const EndpointArgs &a, const EndpointReplay &R, int32_t *mute, const int32_t *ids, int n, cudaStream_t st);
cudaError_t launch_endpoint_clear_muted(const EndpointArgs &a, int32_t *mute, const int32_t *ids, int n, int reset, cudaStream_t st);
cudaError_t launch_endpoint_arm_at(const EndpointArgs &a, const EndpointAt &A, const int32_t *ids, const long long *positions, int n,
                                   cudaStream_t st);
cudaError_t launch_pack_endpointer_rows_muted(const EpRecJob &J, const int32_t *mute, void *records, const int32_t *ids, int n, cudaStream_t st);
cudaError_t launch_unpack_endpointer_rows_muted(const EpRecJob &J, int32_t *mute, const void *records, const int32_t *ids, int n,
                                                cudaStream_t st);
}  // namespace mww

#include "mww_event_positions.h"
namespace mww {
// event positions (mww_event_positions.cu, positions and bodies in mww_event_positions.h; companion library
// libmww_event_positions.so), one launch each.
// the plain detector's update (row_cutoff == nullptr: uniform mode) that also writes positions[slot] for every stored event,
// step t of the call ending at last_end - (n_steps - 1 - t) step_samples
cudaError_t launch_detector_update_at(const DetectorArgs &a, const double *row_cutoff, const float *probs, int n_steps, long long pitch,
                                      long long *positions, long long last_end, long long step_samples, cudaStream_t st);
// the models detector's update that also writes positions[slot], WAKE step j of model k ending at row0_end + hop e_k(j)
cudaError_t launch_detector_models_update_at(const DetectModelsArgs &a, long long *positions, long long row0_end, int hop, cudaStream_t st);
cudaError_t launch_detector_models_update_at(const DetectModelsArgsT<DetectModelRows> &a, long long *positions, long long row0_end, int hop,
                                             cudaStream_t st);
// out [n][out_stride]: row i = samples [ends[i] - n_samples, ends[i]) of stream ids[i] from ring [n_streams][C], `seen` samples
// appended (ids and ends in device memory; zeros outside the ring and for ids outside [0, n_streams))
cudaError_t launch_history_read_at(const int16_t *ring, int C, long long seen, const int32_t *ids, const long long *ends, int n, int n_streams,
                                   int n_samples, int16_t *out, long long out_stride, int sm_count, cudaStream_t st);
// ids [capacity] and ends [capacity]: verify_slot_at of every slot of a timed detector; *count is read on the device
cudaError_t launch_verify_slots_at(const long long *count, const mww_event *events, const long long *positions, int capacity, int model,
                                   long long post, long long seen, int C, int n_samples, int32_t *ids, long long *ends, cudaStream_t st);
}  // namespace mww

#include "mww_detector_groups.h"
namespace mww {
// grouped detection (mww_detector_groups.cu, key, offer and close in mww_detector_groups.h; companion library
// libmww_detector_groups.so).  An update is two launches, the timed update whose grouped rows offer their events to their
// group slots and the close of every slot; a flush is the close alone.
cudaError_t launch_detector_update_grouped(const DetectorArgs &a, const double *row_cutoff, const float *probs, int n_steps, long long pitch,
                                           const GroupArgs &g, long long last_end, long long step_samples, cudaStream_t st);
cudaError_t launch_detector_models_update_grouped(const DetectModelsArgs &a, const GroupArgs &g, long long row0_end, long long row_end, int hop,
                                                  cudaStream_t st);
// per-row mode: the update over per-row descriptors, the close over `base` (the uniform descriptors, for seen and stride)
cudaError_t launch_detector_models_update_grouped(const DetectModelsArgsT<DetectModelRows> &a, const DetectModelsArgs &base, const GroupArgs &g,
                                                  long long row0_end, long long row_end, int hop, cudaStream_t st);
cudaError_t launch_detector_groups_flush(const DetectorArgs &a, const GroupArgs &g, cudaStream_t st);
cudaError_t launch_detector_models_groups_flush(const DetectModelsArgs &a, const GroupArgs &g, cudaStream_t st);
}  // namespace mww

#include "mww_group_arbitration.h"
namespace mww {
// group arbitration (mww_group_arbitration.cu, spans, level, key and close in mww_group_arbitration.h; companion library
// libmww_group_arbitration.so): the grouped launches above with each candidate's level measured at its offer and compared
// first at the close.  The same two launches per update, one per flush.
cudaError_t launch_detector_update_arbitrated(const DetectorArgs &a, const double *row_cutoff, const float *probs, int n_steps, long long pitch,
                                              const GroupArgs &g, const ArbitrationArgs &r, long long last_end, long long step_samples,
                                              cudaStream_t st);
cudaError_t launch_detector_models_update_arbitrated(const DetectModelsArgs &a, const GroupArgs &g, const ArbitrationArgs &r, long long row0_end,
                                                     long long row_end, int hop, cudaStream_t st);
cudaError_t launch_detector_models_update_arbitrated(const DetectModelsArgsT<DetectModelRows> &a, const DetectModelsArgs &base, const GroupArgs &g,
                                                     const ArbitrationArgs &r, long long row0_end, long long row_end, int hop, cudaStream_t st);
cudaError_t launch_detector_arbitrated_flush(const DetectorArgs &a, const GroupArgs &g, const ArbitrationArgs &r, cudaStream_t st);
cudaError_t launch_detector_models_arbitrated_flush(const DetectModelsArgs &a, const GroupArgs &g, const ArbitrationArgs &r, cudaStream_t st);
}  // namespace mww

#include "mww_media_guard.h"
namespace mww {
// media guard (mww_media_guard.cu, bodies in mww_media_guard.h; companion library libmww_media_guard.so), one launch each.
// The slots of a check: a detector's event slots [0, n) when events is set (count, events, positions and ev_group its
// buffers, ev_group nullptr when ungrouped), else the n listed ids ending at ends (households may be nullptr)
struct MediaSlotsArgs {
    int n, n_streams, C, n_samples;
    long long seen;
    const int32_t *ids; const long long *ends; const int32_t *households;
    const long long *count; const mww_event *events; const long long *positions; const int32_t *ev_group;
    int capacity, model; long long post;
};
// [n] each: the slots, each valid slot's rank among them, and the counters the match adds to; state: the guard's ring state
struct MediaSlotsOut {
    int32_t *sid, *rid, *hh, *rank, *count, *clip_hit;
    long long *end, *pos;
    MediaRingState *state;
};
cudaError_t launch_media_slots(const MediaSlotsArgs &a, const MediaSlotsOut &o, cudaStream_t st);
// fp [n][fp_stride]: words [0, words) of each of the n clips whose feature rows are feat [n][rows][40]
cudaError_t launch_media_fingerprint(const uint16_t *feat, long long rows, int n, int words, uint64_t *fp, long long fp_stride, cudaStream_t st);
// the lag search of every valid slot against this check's other valid slots, the ring's entries and the registered clips
struct MediaMatchArgs {
    const uint64_t *fp; int words, n;
    const int32_t *rid, *hh; const long long *pos;
    const uint64_t *ring_fp; const int32_t *ring_stream, *ring_hh; const long long *ring_pos; int ring;
    const MediaRingState *state;
    const uint64_t *clip_fp; const long long *clip_off; const int32_t *clip_len, *clip_task0; int n_clips; long long clip_tasks;
    int max_lag, min_overlap, max_ber_milli; long long window;
    int32_t *count, *clip_hit;
    int tasks_per_cta;
};
size_t media_match_smem(int words);
cudaError_t launch_media_match(const MediaMatchArgs &a, cudaStream_t st);
// matches, media and passed [n] (each may be nullptr) and the ring append
struct MediaDecideArgs {
    int n, words, ring, min_matches;
    const uint64_t *fp; const int32_t *sid, *rid, *hh, *rank, *count, *clip_hit, *confirmed; const long long *pos;
    const MediaRingState *state;
    int32_t *matches, *media, *passed;
    uint64_t *ring_fp; int32_t *ring_stream, *ring_hh; long long *ring_pos;
};
cudaError_t launch_media_decide(const MediaDecideArgs &a, cudaStream_t st);
}  // namespace mww

#include "mww_playback.h"
namespace mww {
// playback guard (mww_playback.cu, bodies in mww_playback.h; companion library libmww_playback.so), one launch each.
// the n_jobs jobs (device memory) of a write call: job j with a row writes row j of audio [.][audio_stride], n_samples each, into
// ring [rows][C] and sets row_of[stream] and head[row]; a job with row -1 sets row_of[stream] = -1
cudaError_t launch_playback_write(const PlaybackJob *jobs, int n_jobs, const int16_t *audio, long long audio_stride, int n_samples,
                                  int16_t *ring, int C, int32_t *row_of, long long *head, cudaStream_t st);
// The slots of a check or a read: a detector's event slots [0, n) when events is set (count, events and positions its buffers),
// else the n listed ids ending at ends.  out [n][out_stride]: row i = pb over [e_i - min_delay - L, e_i - min_delay) of slot i's
// stream; with sid set (a check) also sid and heard [n].  vec is set by the launcher.
struct PlaybackSlotsArgs {
    int n, n_streams, C, L;
    long long seen, min_delay;
    const int32_t *ids; const long long *ends;
    const long long *count; const mww_event *events; const long long *positions;
    int capacity, model; long long post;
    const int16_t *ring; const int32_t *row_of; const long long *head;
    int16_t *out; long long out_stride;
    int32_t *sid, *heard;
    int vec;
};
cudaError_t launch_playback_slots(const PlaybackSlotsArgs &a, cudaStream_t st);
// out_scores, out_flagged and out_passed [n] (each may be nullptr): playback_decide of every slot from the verifier's scores
cudaError_t launch_playback_decide(int n, const int32_t *sid, const int32_t *heard, const float *scores, double cutoff, const int32_t *confirmed,
                                   float *out_scores, int32_t *out_flagged, int32_t *out_passed, cudaStream_t st);
}  // namespace mww
