/*
 * include/mww.h -- C-ABI of libmww_b200.so: the drop-in boundary for microWakeWord's streaming
 * inference hot path on H100 (sm_90a).
 *
 * The reference crosses into native code at three places, all un-vendored third-party libraries
 * (SURVEY.md 2.1); each entry point below names the reference call site it replaces:
 *
 *   microwakeword/inference.py:36-39    tf.lite.Interpreter(model_path) + allocate_tensors()  -> mww_create
 *   microwakeword/inference.py:41-45    get_input_details()/get_output_details()              -> mww_get_info
 *   microwakeword/audio/audio_utils.py:52      MicroFrontend()   (fresh state)               -> mww_reset
 *   microwakeword/audio/audio_utils.py:57-62   MicroFrontend.ProcessSamples(160 samples)     -> mww_features
 *   microwakeword/audio/audio_utils.py:69-81   frontend_op.audio_microfrontend(...)          -> mww_features
 *   microwakeword/inference.py:113-119  set_tensor / invoke / get_tensor, once per 30 ms      -> mww_infer_features
 *   microwakeword/inference.py:66-80    predict_clip (features + predict_spectrogram)         -> mww_predict_clip[_host]
 *   microwakeword/audio/audio_utils.py:47-48   float clip -> int16 (x * 32768, clipped)      -> the *_f32 entry points
 *
 * Conventions
 *   - plain C types only; every d_* pointer is DEVICE memory on the handle's GPU (for PyTorch
 *     callers: tensor.data_ptr()), every h_* pointer is HOST memory.  The caller owns all I/O
 *     buffers; the library owns weights, per-stream state and scratch.
 *   - return 0 on success, a negative MWW_E* code on failure; mww_last_error() gives the message.
 *   - calls are asynchronous on `cu_stream` (a cudaStream_t / CUstream passed as void*, NULL = the
 *     legacy default stream) unless the name ends in _host.  One handle per GPU per host thread.
 *   - a handle carries `n_streams` independent audio streams that advance IN LOCKSTEP: every
 *     stateful call processes all of them with the same number of samples / rows.
 *   - there is no CPU fallback: without a CUDA device mww_create fails with MWW_ECUDA.
 */
#ifndef MWW_H_
#define MWW_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MWW_OK 0
#define MWW_EINVAL (-1)      /* bad argument */
#define MWW_EMODEL (-2)      /* malformed / unsupported model container */
#define MWW_ECUDA (-3)       /* CUDA runtime error (message has the cudaError string) */
#define MWW_ENOMEM (-4)
#define MWW_EUNSUPPORTED (-5)

#define MWW_NUM_FEATURES 40
#define MWW_HOP_SAMPLES 160      /* 10 ms */
#define MWW_WINDOW_SAMPLES 480   /* 30 ms */

/* feature-row element types accepted by mww_infer_features (inference.py:93-96,110) */
#define MWW_ROWS_U16 0   /* raw frontend output; scaled by 0.0390625 on load (inference.py:94) */
#define MWW_ROWS_F32 1   /* already-scaled float features */
#define MWW_ROWS_I8 2    /* pre-quantised int8 rows for a quantised model (inference.py:110) */

typedef struct mww_handle mww_t;

typedef struct mww_info {
    int32_t n_streams;             /* streams carried by the handle */
    int32_t device;
    int32_t is_quantized;          /* inference.py:44 */
    int32_t input_feature_slices;  /* inference.py:45  (= first-conv stride, modes.py:62-63) */
    int32_t num_features;          /* 40 */
    float input_scale;             /* int8 models: quantisation of the input tensor (utils.py:308-313) */
    int32_t input_zero_point;
    float output_scale;            /* int8 models: 1/256 (TFLite LOGISTIC); the reference dequantises with /255 */
    int32_t output_zero_point;
    int32_t state_bytes_per_stream;
    int32_t frontend_buffered;     /* samples currently held in the window carry (0..479) */
    int32_t pending_rows;          /* feature rows waiting for a full stride */
    int32_t sm_count;
    int32_t macs_per_step;
    int32_t hop_samples;           /* samples between feature windows (mww_set_window_step; default 160 = 10 ms) */
} mww_info;

/* Parse an MWW model container (microwakeword_b200/model_file.py), upload the weights to `device`
 * and allocate zeroed state for `n_streams` streams.  model_blob == NULL creates a frontend-only
 * handle (mww_features works, the NN entry points return MWW_EINVAL).  On failure *out is NULL and
 * mww_last_error(NULL) describes why.
 * Architectures: the container's `arch` tensor selects the kernels.  The okay_nabu MixedNet
 * (notebooks/basic_training_notebook.ipynb:503-509) runs on the tensor-core kernels; any other geometry of the
 * reference's default block structure (mixednet.py:278-386 with other --pointwise_filters / --mixconv_kernel_sizes /
 * --first_conv_* / --stride values) runs on the run-time-geometry kernels with the same entry points, state layout
 * rule (first-conv ring, block rings, head ring; oldest row first) and results.  mww_info.input_feature_slices is the
 * model's stride, state_bytes_per_stream its ring state.  A block whose largest MixConv kernel is 1 has no MixConv
 * layer in the reference graph (mixednet.py:346-348); the container carries it as the exact identity depthwise stage
 * (tap 1, bias 0; int8: weight 1, multiplier 1.0, the previous tensor's quantisation) so the block structure stays
 * uniform and results are those of the reference graph.  Topologies outside that family -- repeat_in_block > 1,
 * residual branches (mixednet.py:336-358), pooled / attention heads (:362-381), first_conv_kernel_size < stride --
 * are answered with MWW_EUNSUPPORTED; okay_nabu and the models of esphome/micro-wake-word-models' v2 family use none. */
int mww_create(const void *model_blob, size_t n_bytes, int device, int n_streams, mww_t **out);
int mww_destroy(mww_t *h);
const char *mww_last_error(const mww_t *h);
int mww_get_info(const mww_t *h, mww_info *out);

/* Fresh frontend + zero ring buffers.  ids == NULL (n ignored): all streams, and the lockstep
 * counters (buffered samples, pending rows) return to 0 -- the exact analogue of a new
 * MicroFrontend() / a freshly loaded interpreter.  ids != NULL: h_ids[0..n) streams get zeroed
 * state but keep the shared counters (their history reads as silence) -- this is how a stream joins or
 * leaves a handle that keeps serving the others: a constant number of launches whatever n is, and valid
 * while the rings are rotated by live calls (fresh state is rotation-invariant).
 * mww_reset_device_ids is the same with the id list already in DEVICE memory (e.g. produced by the
 * detection kernels: the streams that just fired); ids outside [0, n_streams) are ignored. */
int mww_reset(mww_t *h, const int32_t *h_ids, int n, void *cu_stream);
int mww_reset_device_ids(mww_t *h, const int32_t *d_ids, int n, void *cu_stream);

/* Fresh frontend only (what a new MicroFrontend() per clip gives the reference, audio_utils.py:52):
 * zero window buffer, zero noise estimates, buffered-sample counter 0.  NN rings are untouched --
 * the reference never resets the interpreter between clips (inference.py:52-64, test.py:335-341). */
int mww_reset_frontend(mww_t *h, void *cu_stream);

/* window_step of the frontend in samples (audio_utils.py:69-81 forwards step_ms to the TF op, whose default on this path is
 * 20 ms = 320 samples; pymicro_features hard-wires 10 ms = 160, the default here).  Any even value in [16, 480]; only while
 * the frontend holds no buffered samples (after create / mww_reset / mww_reset_frontend).  With a hop other than 160 every
 * call runs the run-time-hop kernel (one CTA per stream); the row counts below use this hop in place of 160. */
int mww_set_window_step(mww_t *h, int hop_samples);

/* Frontend only.  d_audio: int16 [n_streams][n_samples] with row pitch `audio_stride` samples.
 * Appends the samples to every stream's window buffer and emits one uint16[40] row per completed
 * 10 ms hop into d_feat [n_streams][max_rows][40].  *h_rows_out = rows emitted per stream
 * ((buffered + n_samples - 480) / 160 + 1 when that is >= 1, else 0).  Does not touch the NN state. */
int mww_features(mww_t *h, const int16_t *d_audio, int n_samples, long long audio_stride,
                 uint16_t *d_feat, int max_rows, int *h_rows_out, void *cu_stream);
/* Same, with float32 audio (nominally in [-1, 1]) in device memory; audio_stride is in samples.  The
 * frontend kernels convert each sample as the reference converts float clips (audio_utils.py:47-48):
 * int16(trunc(clamp(x * 32768, -32768, 32767))) with the product in float32, NaN -> 0.  Results and
 * state are bit-identical to mww_features on the converted samples, and the window buffer holds int16
 * either way, so int16 and float32 calls may alternate on one handle.  Any pointer alignment and
 * pitch work; a 16-byte-aligned buffer whose pitch, n_samples and buffered count are multiples of 8
 * takes the vector loads. */
int mww_features_f32(mww_t *h, const float *d_audio, int n_samples, long long audio_stride,
                     uint16_t *d_feat, int max_rows, int *h_rows_out, void *cu_stream);

/* NN only.  d_rows: [n_streams][n_rows][40] of `row_type`, stream pitch `rows_stride` rows.
 * Rows are appended to the pending rows; every full `input_feature_slices` rows run one model step.
 * d_probs [n_streams][max_probs] receives one probability per step (for a quantised model the
 * uint8 output already divided by 255 as inference.py:162-170 does).  *h_probs_out = steps run. */
int mww_infer_features(mww_t *h, const void *d_rows, int row_type, int n_rows, long long rows_stride,
                       float *d_probs, int max_probs, int *h_probs_out, void *cu_stream);

/* Frontend + NN on device buffers (scratch features stay inside the library). */
int mww_predict_clip(mww_t *h, const int16_t *d_audio, int n_samples, long long audio_stride,
                     float *d_probs, int max_probs, int *h_probs_out, void *cu_stream);
/* Same, with float32 device audio converted inside the frontend kernels (see mww_features_f32):
 * probabilities and state are bit-identical to mww_predict_clip on the converted samples. */
int mww_predict_clip_f32(mww_t *h, const float *d_audio, int n_samples, long long audio_stride,
                         float *d_probs, int max_probs, int *h_probs_out, void *cu_stream);

/* Same, from/to HOST buffers: the library tiles the streams, overlaps the host->device copy of one
 * tile with the kernels of the previous one, and returns when h_probs is complete.  Pinned host
 * memory (mww_host_alloc) gives full-rate copies; pageable memory works too.  The call has no stream
 * argument: it first waits for everything queued on the device so far (cudaDeviceSynchronize), so
 * mww_reset / live calls issued earlier on any stream are ordered before it. */
int mww_predict_clip_host(mww_t *h, const int16_t *h_audio, int n_samples, long long audio_stride,
                          float *h_probs, int max_probs, int *h_probs_out);

/* The audio somewhere else than this GPU's own memory: device memory of a PEER GPU of the box (mapped with
 * mww_ipc_open -- the multi-GPU ingest of BASELINE.json configs[4], "scatter stream batches") or host memory.
 *   n_tiles <= 0: a source this GPU's kernels can address (its own memory, or a peer buffer mapped with mww_ipc_open --
 *                 CUDA reports the mapping device for it) is read IN PLACE by the frontend kernel, i.e. over NVLink for a
 *                 peer buffer (= mww_predict_clip; zero-copy, the right choice while the owner's NVLink egress is not the
 *                 bottleneck); anything else (host memory) goes through the staged pipeline with 16 tiles.
 *   n_tiles  > 0: always the staged pipeline: the streams are cut into n_tiles tiles, this GPU's copy engine pulls tile
 *                 t+1 over NVLink / PCIe into a staging buffer while the kernels of tile t run (frontend AND network, so the
 *                 network's time hides behind the pull -- the right choice when the pull is the bottleneck).
 * Scores are written straight into d_probs on THIS device ([n_streams][max_probs]).  Asynchronous and stream-ordered on
 * cu_stream: the call starts after the work queued on cu_stream so far and cu_stream waits for its last kernel.  If a
 * CUDA call fails half-way the handle is left "poisoned": every stateful entry point fails until
 * mww_reset(h, NULL, 0, stream). */
int mww_predict_clip_remote(mww_t *h, const int16_t *src_audio, int n_samples, long long audio_stride,
                            float *d_probs, int max_probs, int *h_probs_out, int n_tiles, void *cu_stream);

/* Per-stream state snapshot for checkpoint / tests (host buffers, synchronous).
 *   h_carry    int16 [n_streams][480]   window buffer (first `frontend_buffered` samples valid)
 *   h_estimate uint32 [n_streams][40]   noise estimates
 *   h_nn       float [n_streams][4176] (fp32 model) or int8 [n_streams][4176] (quantised): ring buffers,
 *              layer order first-conv, block 0..3, head; each [row][channel], oldest row first
 *   h_pending  float/int8 [n_streams][2][40]
 * NULL pointers are skipped. */
int mww_get_state(mww_t *h, int16_t *h_carry, uint32_t *h_estimate, void *h_nn, void *h_pending);
int mww_set_state(mww_t *h, const int16_t *h_carry, int frontend_buffered, const uint32_t *h_estimate,
                  const void *h_nn, const void *h_pending, int pending_rows);

/* Device-to-device copy of the NN ring state of n streams: stream h_dst_ids[i] of `dst` takes the rings of stream
 * h_src_ids[i] of `src`, for i = 0 .. n-1 in order, asynchronously on cu_stream.  Both handles' rings are first put
 * back into the canonical layout (live calls leave them rotated), so the copy is valid whatever calls came before.
 * Frontend state (window carry, noise estimates) and the lockstep counters are not touched.  dst == src is allowed.
 * MWW_EINVAL when the handles are on different devices, were created from different model containers, either holds
 * pending rows, either is frontend-only, or an id is outside [0, n_streams).  This is how a batched evaluation hands
 * one stream's state to and from a single-stream handle without a host round trip of every stream's state.  Each id
 * pair is one cudaMemcpyAsync (the copies must stay ordered for dst == src), so the call is meant for a few streams;
 * moving the state of many streams at once is what mww_get_state / mww_set_state do. */
int mww_copy_nn_state(mww_t *dst, const int32_t *h_dst_ids, const mww_t *src, const int32_t *h_src_ids, int n, void *cu_stream);

/* ---- detection post-processing (microwakeword/test.py:337-341, :94-137, :364-373) -------------------------
 * Tracks are ragged: track i is d_probs[d_offsets[i] .. d_offsets[i] + d_lengths[i]) (float32 probabilities as
 * produced by mww_infer_features / mww_predict_clip).  All four are stateless and asynchronous on cu_stream.
 *   mww_moving_average       out_i[j] = mean(probs_i[j .. j+window)), written at d_out[d_out_offsets[i] + j]
 *   mww_false_accept_counts  d_counts[i][c] = detections of track i at cutoff c (float64 cutoffs) with the
 *                            reference's cooldown rule, evaluated on the moving average
 *   mww_positive_scores      d_scores[i] = max of the moving average of probs_i[ignore:], NaN if too short
 *   mww_accuracy_counts      the per-track rule of test.py:452-484 (tflite_model_accuracy):
 *                            d_false_accepts[i] = crossings prev <= 0.5 < p at index j with j - last > min_gap, where
 *                            prev and last start at 0 on every track and last = j after each counted crossing;
 *                            d_last_positive[i] = 1 if the track's last probability is > 0.5, else 0 (also for an
 *                            empty track).  Either output may be NULL. */
int mww_moving_average(const float *d_probs, const long long *d_offsets, const int *d_lengths, int n_tracks, int max_length,
                       int window, float *d_out, const long long *d_out_offsets, void *cu_stream);
int mww_false_accept_counts(const float *d_probs, const long long *d_offsets, const int *d_lengths, int n_tracks, int window,
                            const double *d_cutoffs, int n_cutoffs, int ignore_slices_after_accept, int *d_counts, void *cu_stream);
int mww_positive_scores(const float *d_probs, const long long *d_offsets, const int *d_lengths, int n_tracks, int window,
                        int ignore_slices_after_accept, float *d_scores, void *cu_stream);
int mww_accuracy_counts(const float *d_probs, const long long *d_offsets, const int *d_lengths, int n_tracks, int min_gap,
                        int *d_false_accepts, int *d_last_positive, void *cu_stream);

/* Per-kernel device timing for roofline reporting.  While enabled, every launch of the four kernel
 * classes is bracketed by CUDA events on the launching stream.  mww_profile_read synchronises the
 * device, adds the elapsed milliseconds into ms[4] and the launch counts into counts[4]
 * (index 0 spectral K1, 1 temporal K2, 2 MixedNet, 3 window-carry update) and clears the record. */
int mww_profile_enable(mww_t *h, int on);
int mww_profile_read(mww_t *h, double *ms4, long long *counts4);

/* Tile timeline of the most recent staged call (mww_predict_clip_host / mww_predict_clip_remote from a peer or host
 * source) made while profiling was enabled: for tile t, ms[4 t + 0..3] = copy start, copy end, kernels start, kernels end,
 * in milliseconds after tile 0's copy start (CUDA events on the library's copy and compute streams; -1 where an event
 * could not be read).  *n_tiles = tiles the call used; at most max_tiles are written.  Synchronises the device and clears
 * the record.  This is what DESIGN.md section 5's per-rank ingest timelines are made of. */
int mww_timeline_read(mww_t *h, float *ms, int max_tiles, int *n_tiles);

/* Kernel launches issued by this handle since creation (bench.py's gpu_launches). */
long long mww_launch_count(const mww_t *h);

/* Stream-ordered device copy issued on the CALLER'S stream: cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, cu_stream).
 * Used by the multi-GPU ingest (bench.py's pull-only probe and equality checks; the north_star's "scatter stream batches"):
 * `src` may be peer memory of another GPU of the box mapped through CUDA IPC, and because the stream belongs to the
 * DESTINATION device the transfer is a copy-engine pull inside the caller's own context -- no communication kernel and
 * no work in a second context on the source GPU.  The reference has no counterpart (it is single-process, SURVEY.md 2.2).
 * Returns 0 or a negative MWW_ECUDA; no handle is involved (the message goes to mww_last_error(NULL)). */
int mww_copy_async(void *d_dst, const void *d_src, size_t bytes, void *cu_stream);

/* CUDA IPC for the multi-GPU ingest buffer, opened in the CALLER'S device context (sharding.py::IngestBuffer).
 * mww_ipc_alloc: cudaMalloc on `device` + cudaIpcGetMemHandle (64 opaque bytes to hand to the other ranks of the box).
 * mww_ipc_open: cudaIpcOpenMemHandle(..., cudaIpcMemLazyEnablePeerAccess) with `device` (the OPENING rank's own GPU)
 * current, so the mapping lives in that rank's context and the rank never creates a context on the exporting GPU --
 * torch's tensor rebuild opens the handle under the exporter's device index instead, which leaves one extra context per
 * peer on the ingest GPU (DESIGN.md section 5, the 8-GPU ingest).  mww_ipc_close / mww_ipc_free undo them.
 * All return 0 or a negative MWW_ECUDA / MWW_EINVAL; the message goes to mww_last_error(NULL). */
int mww_ipc_alloc(size_t bytes, int device, void **d_ptr, unsigned char *handle64);
int mww_ipc_open(const unsigned char *handle64, int device, void **d_ptr);
int mww_ipc_close(void *d_ptr, int device);
int mww_ipc_free(void *d_ptr, int device);

/* Pinned host memory placed on the NUMA node the GPU hangs off (/sys/bus/pci/devices/<bdf>/numa_node): the calling
 * thread is moved to that node's CPUs (and MPOL_PREFERRED set, where the container allows it) for the duration of the
 * cudaHostAlloc, then put back.  On a two-socket 8-GPU box the default placement puts every rank's buffer on the node
 * the process happened to start on and the GPUs of the other socket copy across the inter-socket link, which lowers
 * every such rank's host->device rate.  *numa_node_out (optional) = the node, -1 when
 * the topology cannot be read (then this is a plain cudaHostAlloc).  mww_bind_host_thread moves the CALLING thread to
 * the GPU's node for good (a rank calls it once, before anything else allocates). */
int mww_host_alloc(size_t bytes, int device, void **h_ptr, int *numa_node_out);
/* Same, write-combined (cudaHostAllocWriteCombined): for INPUT buffers the CPU only writes (sequentially) and the GPU only
 * reads -- audio on its way to mww_predict_clip_host.  Transfers of write-combined memory are not snooped on the PCIe bus;
 * CPU reads of it are very slow, so never use it for the probability buffer.  Freed with mww_host_free. */
int mww_host_alloc_wc(size_t bytes, int device, void **h_ptr, int *numa_node_out);
int mww_host_free(void *h_ptr);
int mww_bind_host_thread(int device, int *numa_node_out);

#ifdef __cplusplus
}
#endif
#endif /* MWW_H_ */
