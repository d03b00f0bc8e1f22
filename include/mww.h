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
 *   (telephony: G.711 mu-law / A-law bytes, decoded on the GPU)                             -> the *_g711 entry points
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
 * are answered with MWW_EUNSUPPORTED; okay_nabu and the models of esphome/micro-wake-word-models' v2 family use none.
 * Hybrid models: an fp32 container with `hy/mode` (the float .tflite the reference writes with quantize=False, whose
 * large conv / depthwise / dense weights the converter stores as per-channel int8) runs TFLite's hybrid arithmetic --
 * each such op quantises its float input to int8 on every step -- on the run-time-geometry hybrid kernel, whatever the
 * architecture, okay_nabu's included.  It reads as an fp32 model everywhere (mww_info.is_quantized 0, float rows and
 * probabilities, fp32 ring state in the layout above). */
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

/* ---- Input sample rate ----------------------------------------------------------------------------------------------
 * A handle takes audio at one input rate, 16000 Hz unless mww_set_input_rate says otherwise: 8000, 22050, 24000, 32000,
 * 44100 or 48000 Hz (L / M = 16000 / rate in lowest terms: 2/1, 320/441, 2/3, 1/2, 160/441, 1/3).  At any rate but 16000 a
 * resampler kernel turns each stream tile's samples into 16 kHz int16 samples before the frontend, one launch per tile;
 * at 16000 nothing changes.  Every audio entry point then takes n_samples AT THE INPUT RATE (float32 audio is first
 * converted to int16 as everywhere else); rows and model steps follow from the 16 kHz count the call yields.
 *
 * The resampler is defined in integers.  Taps h[0, N): a Kaiser-windowed sinc designed in double (scipy.signal.kaiserord
 * for 80 dB attenuation over the transition band, length made odd; scipy.signal.firwin with cutoff at the band's centre,
 * unit DC gain), times L, in Q15, rounded and clamped to int16.  Decimating rates pass to 7 500 Hz and stop from 8 500 Hz
 * (the mel filterbank ends at 7 500 Hz, so whatever folds back stays above every feature); 8 kHz passes to 3 600 Hz and
 * stops from 4 400 Hz.  After Q15 rounding the stopband is at least 70 dB down at every rate (72.8 dB at 32 kHz, 70.4 dB
 * at 48 kHz, where the 243 taps are shortest) and the passband ripple is within 0.0004.  Output n is
 *     y[n] = sat16((sum_j h[j] x_up[n M - j] + 2^14) >> 15),   x_up = the input zero-stuffed by L,
 * scipy.signal.upfirdn(h, x, L, M) followed by the rounding shift, computed exactly.  Calls concatenate exactly: after N
 * input samples a stream has been given ceil(N L / M) 16 kHz samples, the prefix of one upfirdn over all of its input.
 * Each stream keeps the last H = ceil(N_taps / L) input samples as history; one counter of input samples seen belongs to
 * the handle (all streams advance in lockstep).  A 30 ms call (e.g. 1 440 samples at 48 kHz, 1 323 at 44.1 kHz) yields
 * 480 samples and takes the live-step kernels.  One call must keep n_samples * L below 2^31 (MWW_EINVAL otherwise).
 *
 * mww_reset(NULL) and mww_reset_frontend zero the history and the counter; mww_reset(ids) / mww_reset_device_ids zero
 * those streams' history.  mww_export_streams / mww_import_streams return MWW_EUNSUPPORTED on a handle whose rate is not
 * 16000 (the records have no room for the history); mww_export_resampled_streams / mww_import_resampled_streams carry it
 * (see "moving resampled streams" below).  The staged paths tile input-rate audio; the 16 kHz tile scratch counts against
 * MWW_SCRATCH_MB. */
/* Allowed when mww_set_window_step is (no buffered samples) and the counter is 0; any hop.  A rate outside the list:
 * MWW_EUNSUPPORTED; buffered samples: MWW_EINVAL.  Either way the handle is unchanged. */
int mww_set_input_rate(mww_t *h, int rate);
/* *rate = the input rate, *inputs_seen = input samples every stream has been given since the last reset (0 at 16000) */
int mww_get_input_rate(const mww_t *h, int *rate, long long *inputs_seen);
/* history int16 [n_streams][H] (may be NULL) and the counter; at 16000 there is no history and the counter is 0.  Set
 * synchronises the device; a negative counter (or a non-zero one at 16000) is MWW_EINVAL. */
int mww_get_resampler_state(mww_t *h, int16_t *h_history, long long *inputs_seen);
int mww_set_resampler_state(mww_t *h, const int16_t *h_history, long long inputs_seen);
/* The taps of `rate` without a handle or a GPU: *n_taps, *L, *M (each may be NULL), and the taps (int16 values) in
 * out[0, n_taps) when max_taps >= n_taps.  16000: n_taps = 0.  A rate outside the list: MWW_EUNSUPPORTED. */
int mww_resample_taps(int rate, int32_t *out, int max_taps, int *n_taps, int *L, int *M);

/* ---- Per-stream input rates ------------------------------------------------------------------------------------------
 * A handle in per-stream-rate mode gives each stream s its own rate r_s from the list above (L_s / M_s = 16000 / r_s), so
 * one handle serves telephony, files and WebRTC at once.  The handle keeps one lockstep counter t: the 16 kHz samples every
 * stream has been given since the last full reset.  Every audio call names its length n16 in 16 kHz samples, passed as
 * n_samples; n16 must be even (an 8 kHz stream yields 16 kHz samples in pairs), 0 included.  Row s of the caller's audio
 * holds the stream's next
 *     D_s = N(t + n16, r_s) - N(t, r_s)   input samples,   N(t, r) = floor(t M / L)   (mww_rate_inputs),
 * and the call advances t by n16.  The N identity: for even t, ceil(N(t, r) L / M) = t at every rate.  Proof: write
 * t M = N L + rho with 0 <= rho < L, so N L <= t M.  At 8 kHz (L = 2, M = 1) rho = t mod 2 = 0, so N L = t M.  At every
 * other rate M >= L > rho, so N L > t M - M.  Either way (t - 1) M < N L <= t M.  After N(t, r_s) inputs the causal rule
 * above has therefore emitted exactly t samples at 16 kHz, and every call gives every stream n16 of them.  A 30 ms call is
 * n16 = 480 at every rate: 240 / 480 / 720 / 960 / 1 323 / 1 440 samples at 8 / 16 / 24 / 32 / 44.1 / 48 kHz, and 661 or
 * 662 in turn at 22.05 kHz.
 *
 * Stream s is bit-identical to a stream of a handle at the single rate r_s (a plain 16 kHz handle when r_s = 16000) given
 * the same D_s samples in every call: features, every model's probabilities and state, and its resampler history.
 * Changing a stream's rate zeroes its resampler history and nothing else: it then continues as a stream at the new rate
 * that has been given N(t, r_new) samples of silence.  Call mww_reset(ids) as well to restart its frontend and models.
 *
 * In this mode every audio entry point (mww_features*, mww_predict_clip*, host, remote, _multi, _f32, _g711) reads n_samples as
 * n16; an odd n16, or an audio_stride below the call's largest D_s, is MWW_EINVAL before any work.  Each tile runs one
 * resampler launch per rate with streams in it, on those streams only; 16 kHz streams are copied.  mww_get_input_rate
 * reports MWW_RATE_PER_STREAM and t.  mww_get_resampler_state / mww_set_resampler_state move history
 * int16 [n_streams][H_max] and t, H_max = 243 (the largest H of any rate; 52, 111, 122, 163, 222 and 243 at 8, 22.05, 24,
 * 32, 44.1 and 48 kHz): each stream uses the first H of its own rate, and set refuses an odd t.  mww_reset(NULL) and
 * mww_reset_frontend zero every history and t and keep the rates; mww_reset(ids) zeroes those streams' histories.
 * mww_export_streams / mww_import_streams return MWW_EUNSUPPORTED; mww_export_resampled_streams and
 * mww_import_resampled_streams move these streams.  mww_set_input_rate(h, r), allowed at t = 0, returns the handle to one
 * rate for every stream. */
#define MWW_RATE_PER_STREAM 0
/* Rate h_rates[i] for stream h_ids[i].  The first call puts the handle into per-stream-rate mode, with every stream not
 * listed at 16000; it is allowed only where mww_set_input_rate is (no buffered samples, counter 0) and on a 16 kHz handle
 * (MWW_EINVAL otherwise).  Later calls are allowed wherever a stateful call is.  Ordered on cu_stream; the listed streams'
 * histories are zeroed, whether their rate changes or not.  A rate outside the list: MWW_EUNSUPPORTED; an id out of range
 * or listed twice, or n < 0: MWW_EINVAL.  Every refusal leaves the handle unchanged. */
int mww_set_stream_rates(mww_t *h, const int32_t *h_ids, const int32_t *h_rates, int n, void *cu_stream);
/* h_rates [n_streams] (may be NULL): each stream's rate, the handle's rate for every stream on a single-rate handle.
 * *samples16_seen (may be NULL): t; on a single-rate handle the 16 kHz samples its resampler has emitted (0 at 16000). */
int mww_get_stream_rates(const mww_t *h, int32_t *h_rates, long long *samples16_seen);
/* *inputs = N(samples16, rate) = floor(samples16 M / L), without a handle or a GPU.  A rate outside the list:
 * MWW_EUNSUPPORTED; samples16 outside [0, 2^50] or inputs NULL: MWW_EINVAL. */
int mww_rate_inputs(int rate, long long samples16, long long *inputs);

/* ---- Per-stream sample formats -----------------------------------------------------------------------------------------
 * A handle with per-stream rates also gives each stream s a sample format f_s, so that telephony (G.711 bytes at 8 kHz) and
 * WebRTC or satellites (int16 or float32) feed one handle in one call.  Four formats, one code each (the G.711 codes are
 * those of MWW_G711_ULAW / MWW_G711_ALAW below):
 *     MWW_FORMAT_S16 (0) int16 PCM, 2 bytes;   MWW_FORMAT_ULAW (1) mu-law, 1 byte;   MWW_FORMAT_ALAW (2) A-law, 1 byte;
 *     MWW_FORMAT_F32 (3) float32 in [-1, 1], 4 bytes, converted as mww_features_f32 converts it.
 * Every stream starts as MWW_FORMAT_S16.  The _mixed entry points (mww_features_mixed, mww_predict_clip_mixed and the
 * _multi, _host, _host_multi, _remote and _remote_multi forms) take the arguments of their _f32 counterparts with the audio
 * as bytes.  Row s of the audio starts at audio + s * audio_stride, audio_stride in BYTES, and holds the stream's
 *     D_s * bytes(f_s)   bytes   (D_s as above: the call's input samples of stream s at its rate),
 * its samples in its own format; the bytes after them, up to the next row, are never read.  audio_stride must be at least the
 * largest such row of any (rate, format) pair present on the handle, and the base address and audio_stride must both be
 * multiples of 4 (float rows aligned); n_samples is n16 as in every call of this mode.  Anything else is MWW_EINVAL before
 * any work, and a handle without per-stream rates is MWW_EUNSUPPORTED; either way the handle is unchanged.
 * Stream s is bit-identical to the same stream given its samples decoded to int16 (the G.711 rule below, or the float32
 * conversion) in an int16 call: features, every model's probabilities and state, resampler history and audio history.  The
 * resampler decodes each row on load, one launch per rate with streams in the tile as for int16 rows (16 kHz streams on its
 * identity plan), and every later kernel reads its 16 kHz int16 output.  The staged paths copy each tile's rows as wide as
 * the tile's widest row, rounded up to 4 bytes: a caller that gives neighbouring streams like sources moves one byte per
 * G.711 sample.  Their two staging tiles count against MWW_SCRATCH_MB.  A single-rate handle has no per-stream formats; its
 * calls take one sample type for every row (int16, _f32, _g711). */
#define MWW_FORMAT_S16 0
#define MWW_FORMAT_ULAW 1
#define MWW_FORMAT_ALAW 2
#define MWW_FORMAT_F32 3
/* Format h_formats[i] for stream h_ids[i], ordered on cu_stream.  A format changes no state: decoding is memoryless and the
 * resampler history holds decoded int16 samples.  A handle without per-stream rates: MWW_EUNSUPPORTED; an unknown code, an id
 * out of range or listed twice, or n < 0: MWW_EINVAL.  Every refusal leaves the handle unchanged.  mww_set_input_rate (back
 * to one rate) forgets the formats; mww_set_stream_rates and resets keep them. */
int mww_set_stream_formats(mww_t *h, const int32_t *h_ids, const int32_t *h_formats, int n, void *cu_stream);
/* h_formats [n_streams]: each stream's format (MWW_FORMAT_S16 for every stream of a single-rate handle) */
int mww_get_stream_formats(const mww_t *h, int32_t *h_formats);
int mww_features_mixed(mww_t *h, const uint8_t *d_audio, int n_samples, long long audio_stride,
                       uint16_t *d_feat, int max_rows, int *h_rows_out, void *cu_stream);
int mww_predict_clip_mixed(mww_t *h, const uint8_t *d_audio, int n_samples, long long audio_stride,
                           float *d_probs, int max_probs, int *h_probs_out, void *cu_stream);
int mww_predict_clip_multi_mixed(mww_t *h, const uint8_t *d_audio, int n_samples, long long audio_stride,
                                 float *const *d_probs, const int *max_probs, int *h_probs_out, void *cu_stream);
int mww_predict_clip_host_mixed(mww_t *h, const uint8_t *h_audio, int n_samples, long long audio_stride,
                                float *h_probs, int max_probs, int *h_probs_out);
int mww_predict_clip_host_multi_mixed(mww_t *h, const uint8_t *h_audio, int n_samples, long long audio_stride,
                                      float *const *h_probs, const int *max_probs, int *h_probs_out);
int mww_predict_clip_remote_mixed(mww_t *h, const uint8_t *src_audio, int n_samples, long long audio_stride,
                                  float *d_probs, int max_probs, int *h_probs_out, int n_tiles, void *cu_stream);
int mww_predict_clip_remote_multi_mixed(mww_t *h, const uint8_t *src_audio, int n_samples, long long audio_stride,
                                        float *const *d_probs, const int *max_probs, int *h_probs_out, int n_tiles, void *cu_stream);

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

/* mww_predict_clip_host / mww_predict_clip_remote with float32 audio (nominally in [-1, 1]; audio_stride in samples): the
 * staged pipeline copies the float samples as they are, and the frontend kernels convert them on the GPU as
 * mww_features_f32 does.  Probabilities and state are bit-identical to the int16 call on the converted samples, and int16
 * and float32 calls may alternate on one handle.  Ordering, poisoning on a half-way failure and the n_tiles rule are those
 * of the int16 calls; a source this GPU can address with n_tiles <= 0 is read in place (= mww_predict_clip_f32).  Each
 * staging tile holds twice the bytes of an int16 one, so the two float staging tiles count against the scratch budget
 * (MWW_SCRATCH_MB, default 2048): a tile takes at most budget / (2 * 4 * n_samples + the per-stream scratch) streams. */
int mww_predict_clip_host_f32(mww_t *h, const float *h_audio, int n_samples, long long audio_stride,
                              float *h_probs, int max_probs, int *h_probs_out);
int mww_predict_clip_remote_f32(mww_t *h, const float *src_audio, int n_samples, long long audio_stride,
                                float *d_probs, int max_probs, int *h_probs_out, int n_tiles, void *cu_stream);

/* ---- several models over one frontend ---------------------------------------------------------------------------
 * A deployment that listens for several wake words (and a VAD model) on the same audio runs one frontend and K models on
 * its rows.  mww_create_multi makes a handle that carries K >= 1 models of any kind the containers describe (fp32
 * okay_nabu, int8, other geometries and strides, hybrid) over ONE shared frontend: one window carry, one set of noise
 * estimates, one buffered-sample counter and one hop; each model has its own weights, ring state, pending rows and stride.
 * Each predict call runs the frontend once per stream tile and every model on that tile's rows, and on the staged paths
 * copies each audio tile once.  Model k's probabilities, state and pending rows are bit-identical to those of a
 * one-model handle of the same container given the same calls; the frontend state is that of any of them.
 *   - mww_create_multi: blobs[k] / n_bytes[k] for k in [0, n_models), 1 <= n_models <= 64.  A model that fails to load
 *     fails the create; mww_last_error(NULL) starts with "model <k>: ".  mww_create(blob, ...) is the K = 1 case.
 *   - mww_model_count: K (0 for a frontend-only handle).  mww_get_model_info: model k's stride (input_feature_slices),
 *     quantisation, state_bytes_per_stream, pending_rows and macs_per_step; the frontend fields are the shared ones.
 *     mww_get_info reports model 0.
 *   - the _multi predict calls take the arguments of their one-model counterparts with K output buffers: d_probs[k]
 *     [n_streams][max_probs[k]], and h_probs_out[k] (may be NULL) = steps model k ran, which differ between models of
 *     different strides or pending rows.  Every model's buffer is checked before anything is launched.  A 480-sample
 *     call runs each okay_nabu model's live-step kernel (each model's rings rotate on their own).  The staged paths
 *     (_host_multi, _remote_multi) poison the whole handle on a half-way failure, as their one-model counterparts do.
 *   - mww_get_model_state / mww_set_model_state: model k's h_nn / h_pending in the layout of mww_get_state (with model
 *     k's state_bytes_per_stream and stride - 1 pending rows) and its pending_rows counter; NULL pointers are skipped.
 *   - mww_reset (all or by id), mww_reset_device_ids reset the frontend and every model; mww_reset_frontend,
 *     mww_set_window_step and mww_features act on the shared frontend; mww_launch_count and mww_profile_* count every
 *     model's launches.
 *   - on a handle with K > 1, mww_predict_clip[_f32/_host/_remote/_host_f32/_remote_f32], mww_infer_features and
 *     mww_copy_nn_state return MWW_EINVAL, as do mww_get_state / mww_set_state given NN arrays or a nonzero pending_rows (called with those NULL /
 *     0 they read / write the frontend state only): each would advance or replace state for one model only. */
int mww_create_multi(const void *const *blobs, const size_t *n_bytes, int n_models, int device, int n_streams, mww_t **out);
int mww_model_count(const mww_t *h);
int mww_get_model_info(const mww_t *h, int k, mww_info *out);
int mww_predict_clip_multi(mww_t *h, const int16_t *d_audio, int n_samples, long long audio_stride,
                           float *const *d_probs, const int *max_probs, int *h_probs_out, void *cu_stream);
int mww_predict_clip_multi_f32(mww_t *h, const float *d_audio, int n_samples, long long audio_stride,
                               float *const *d_probs, const int *max_probs, int *h_probs_out, void *cu_stream);
int mww_predict_clip_host_multi(mww_t *h, const int16_t *h_audio, int n_samples, long long audio_stride,
                                float *const *h_probs, const int *max_probs, int *h_probs_out);
int mww_predict_clip_remote_multi(mww_t *h, const int16_t *src_audio, int n_samples, long long audio_stride,
                                  float *const *d_probs, const int *max_probs, int *h_probs_out, int n_tiles, void *cu_stream);
int mww_predict_clip_host_multi_f32(mww_t *h, const float *h_audio, int n_samples, long long audio_stride,
                                    float *const *h_probs, const int *max_probs, int *h_probs_out);
int mww_predict_clip_remote_multi_f32(mww_t *h, const float *src_audio, int n_samples, long long audio_stride,
                                      float *const *d_probs, const int *max_probs, int *h_probs_out, int n_tiles, void *cu_stream);
int mww_get_model_state(mww_t *h, int k, void *h_nn, void *h_pending);
int mww_set_model_state(mww_t *h, int k, const void *h_nn, const void *h_pending, int pending_rows);

/* ---- G.711 audio -------------------------------------------------------------------------------------------------
 * Telephony audio arrives as G.711: RTP payload types 0 (PCMU, mu-law) and 8 (PCMA, A-law), or WAV format tags 7 and 6.
 * Each sample is one byte, and the frontend kernels (and the resampler kernel, at any input rate but 16000) decode it on
 * load, so a telephony server sends the bytes as they came: no decode on the host, half the bytes of int16 over PCIe.
 * The rule is ITU-T G.711 as written in the Sun g711.c reference code (Python's audioop, SoX and FFmpeg decode the same):
 *   mu-law: u = ~code & 0xFF; t = ((u & 0x0F) << 3) + 0x84; t <<= (u & 0x70) >> 4;
 *           pcm = (u & 0x80) ? 0x84 - t : t - 0x84                    (range +-32124; codes 0xFF and 0x7F both give 0)
 *   A-law:  a = code ^ 0x55; t = (a & 0x0F) << 4; seg = (a & 0x70) >> 4;
 *           t = seg == 0 ? t + 8 : seg == 1 ? t + 0x108 : (t + 0x108) << (seg - 1);
 *           pcm = (a & 0x80) ? t : -t                                  (range +-32256)
 * Each _g711 entry point takes the arguments of its _f32 counterpart, with the audio as bytes and `law` (MWW_G711_ULAW or
 * MWW_G711_ALAW) right after the audio pointer; audio_stride is in samples, which here are bytes.  Results and state are
 * bit-identical to the int16 call on the decoded samples, and int16, float32, mu-law and A-law calls may alternate on one
 * handle: the window carry and the resampler history hold int16 whatever the input.  Every rule of the counterpart holds
 * unchanged: per-stream rates (n_samples is n16, row s holds D_s bytes), the refusals of the one-model calls on a handle
 * with K > 1 models or stream sets, the n_tiles rule and in-place reads, ordering and poisoning on a half-way staged
 * failure.  A law other than the two is MWW_EINVAL before any device work, with the handle unchanged.  Any pointer alignment
 * and pitch work; an 8-byte-aligned buffer whose pitch, n_samples and buffered count are multiples of 8 takes the vector
 * loads (8 bytes at a time).  A staging tile holds half the bytes of an int16 one, so the staged paths need no staging or
 * scratch beyond what an int16 call uses.  One call's rows share one law. */
#define MWW_G711_ULAW 1
#define MWW_G711_ALAW 2
int mww_features_g711(mww_t *h, const uint8_t *d_audio, int law, int n_samples, long long audio_stride,
                      uint16_t *d_feat, int max_rows, int *h_rows_out, void *cu_stream);
int mww_predict_clip_g711(mww_t *h, const uint8_t *d_audio, int law, int n_samples, long long audio_stride,
                          float *d_probs, int max_probs, int *h_probs_out, void *cu_stream);
int mww_predict_clip_host_g711(mww_t *h, const uint8_t *h_audio, int law, int n_samples, long long audio_stride,
                               float *h_probs, int max_probs, int *h_probs_out);
int mww_predict_clip_remote_g711(mww_t *h, const uint8_t *src_audio, int law, int n_samples, long long audio_stride,
                                 float *d_probs, int max_probs, int *h_probs_out, int n_tiles, void *cu_stream);
int mww_predict_clip_multi_g711(mww_t *h, const uint8_t *d_audio, int law, int n_samples, long long audio_stride,
                                float *const *d_probs, const int *max_probs, int *h_probs_out, void *cu_stream);
int mww_predict_clip_host_multi_g711(mww_t *h, const uint8_t *h_audio, int law, int n_samples, long long audio_stride,
                                     float *const *h_probs, const int *max_probs, int *h_probs_out);
int mww_predict_clip_remote_multi_g711(mww_t *h, const uint8_t *src_audio, int law, int n_samples, long long audio_stride,
                                       float *const *d_probs, const int *max_probs, int *h_probs_out, int n_tiles, void *cu_stream);

/* ---- each model on its own streams ------------------------------------------------------------------------------
 * A server whose satellites each listen for their own wake word runs one frontend over all streams and each model only on
 * the streams that asked for it.  Model k of a handle has a STREAM SET: a strictly increasing list of n_k stream ids in
 * [0, n_streams), 0 <= n_k <= n_streams; the default (mww_create_multi, ids[k] == NULL) is all streams.
 *   - model k's ring state, pending rows and probabilities cover its own streams only, in list order: row j of d_probs[k] /
 *     h_probs[k] ([n_k][max_probs[k]]) belongs to stream ids_k[j].  The buffer of a model with n_k = 0 may be NULL.  The
 *     state is allocated for the n_k members only.
 *   - the frontend still runs once per stream tile over all n_streams streams, and the lockstep counters (buffered samples,
 *     each model's pending rows and ring rotation) are those of a handle without stream sets: the step counts
 *     h_probs_out[k] reports do not depend on n_k.
 *   - bit identity: for every member stream, model k's probabilities and state row are bit-identical to those of the same
 *     stream in a handle where model k covers all streams, given the same calls.
 *   - a model whose members in a stream tile are consecutive stream ids (all streams, or one block) reads that tile's
 *     feature rows in place, with the launches of a handle without stream sets; any other set costs one row-gather launch
 *     per model per tile, into a buffer that counts against MWW_SCRATCH_MB.
 *   - mww_set_model_streams replaces model k's set (h_ids == NULL: all streams), stream-ordered on cu_stream and allowed
 *     wherever a stateful call is (rotated rings and pending rows included).  Streams in both sets keep their ring and
 *     pending-row state exactly; streams that join get the model's fresh state (what mww_reset(ids) gives them: zero rings
 *     for fp32 and hybrid, zero points for int8, zero pending rows); streams that leave lose it.  The frontend is not
 *     touched.  The call returns once the old state is freed (it synchronises cu_stream).  Ids out of range, unsorted or
 *     duplicate ids, n < 0 or a bad k: MWW_EINVAL before any device work, the handle unchanged.
 *   - mww_reset(ids) / mww_reset_device_ids take GLOBAL stream ids: they reset those streams' frontend and, for each model,
 *     the listed streams that are members of it (non-members are ignored for that model).
 *   - mww_get_model_state / mww_set_model_state move [n_k][state elements] / [n_k][stride - 1][40], in list order.
 *     mww_get_model_info reports n_streams = n_k; mww_get_info keeps the handle's n_streams.
 *   - the one-model entry points (mww_predict_clip*, mww_infer_features, mww_copy_nn_state, mww_get_state / mww_set_state
 *     with NN arrays) return MWW_EINVAL on any handle where a model's set is not all streams, K = 1 included: they move
 *     [n_streams]-shaped NN buffers.  The _multi calls are the interface for stream sets. */
/* K models over one frontend, model k only on streams ids[k][0 .. n_ids[k]) (strictly increasing; ids == NULL or
 * ids[k] == NULL: all streams).  State is allocated per model for its own streams only: this is what keeps K models on a
 * large handle within device memory. */
int mww_create_multi_streams(const void *const *blobs, const size_t *n_bytes, int n_models, int device, int n_streams,
                             const int32_t *const *ids, const int *n_ids, mww_t **out);
/* Replace model k's stream set (h_ids == NULL: all streams); stream-ordered on cu_stream, rules above. */
int mww_set_model_streams(mww_t *h, int k, const int32_t *h_ids, int n, void *cu_stream);
/* Model k's stream ids; *n_out = n_k, at most max_ids written. */
int mww_get_model_streams(const mww_t *h, int k, int32_t *h_ids, int max_ids, int *n_out);

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

/* ---- moving streams between handles -------------------------------------------------------------------------------
 * A handle serves a fixed number of streams.  A server that grows or compacts a handle, rebalances streams across the GPUs
 * of a box or checkpoints some streams moves them as STREAM RECORDS: everything one stream carries (frontend and every
 * model), packed on the device by mww_export_streams and written into another handle by mww_import_streams, in a number of
 * launches that does not depend on how many streams move.  The state arrives bit-exact, and a stream that moves continues
 * bit for bit as if it had stayed wherever the arithmetic does not depend on the ring rotation: int8, hybrid and
 * run-time-geometry models, every clip call, and fp32 okay_nabu live calls when the destination's rings are at the
 * rotation the stream left (the same number of live calls since the last clip call, modulo each ring's length).  The
 * fp32 live-step kernel adds a ring's taps in physical row order, so at another rotation the last bits may differ.
 *   - one record, record_bytes long (a multiple of 16), every part padded to 16 bytes:
 *         uint64  member_mask          bit k set: the stream was a member of model k and slot k holds its state
 *         int16   carry[480]           window buffer (first frontend_buffered samples valid)
 *         uint32  estimate[40]         noise estimates
 *         for each model k, in order:  nn[state elements of model k]  float32 or int8, the layout of mww_get_model_state:
 *                                                                     rings CANONICAL, oldest row first
 *                                      pending[max(stride_k - 1, 1)][40]  float32 or int8
 *     d_records is [n][record_bytes], 16-byte aligned, in memory the handle's GPU can address: its own, or a peer buffer
 *     mapped with mww_ipc_open (read or written in place over NVLink).  Between GPUs without a mapping: export on the
 *     source GPU and pull the buffer with mww_copy_async.
 *   - the lockstep counters belong to the handle, not to a stream: they travel beside the records in mww_stream_layout,
 *     which mww_export_streams fills (out may be NULL) and mww_import_streams checks.  mww_stream_layout_get gives a
 *     handle's own layout and current counters without device work (record_bytes sizes the buffer).
 *   - both calls are asynchronous and stream-ordered on cu_stream and take GLOBAL stream ids from host memory, in any
 *     order; export allows an id to appear twice, import refuses it.  n == 0 launches nothing and still fills / checks the
 *     layout.
 *   - mww_export_streams does not change the handle, not even the rotation live calls leave its rings in: the pack kernel
 *     reads each ring row where it lies and writes it oldest first.  For a model the stream is not a member of, its mask
 *     bit is clear and its slot is zero.
 *   - mww_import_streams overwrites exactly the listed streams' state and leaves every other stream's bytes untouched; it
 *     writes each ring at the destination's own rotation, so the two handles may have made different numbers of live
 *     calls.  Per model k: a destination stream that is not a member ignores slot k; a member whose mask bit is set takes
 *     the state; a member whose bit is clear gets the model's fresh state (what mww_reset(ids) and mww_set_model_streams
 *     give: zero rings for fp32 and hybrid, zero points for int8).  Import lowers model k's rows_are_features flag
 *     to the records' for every model with members, whatever the streams listed.
 *   - import is refused with MWW_EINVAL, before any device work and with the handle unchanged, when the records do not fit
 *     the destination: n_models, a model (container, precision, state size), record_bytes, hop_samples, frontend_buffered
 *     or a model's pending_rows differs -- the message names the first such field -- or an id is out of range or listed
 *     twice.  The counters must match because a handle's streams advance in lockstep; two handles that serve 480-sample
 *     live calls always match (320 buffered samples, a constant pending-row count).
 *   - rows_are_features[k] says whether model k's carried first-conv rows are exact feature rows, which is what lets the
 *     fp16 first conv of the okay_nabu clip kernel run; import lowers the destination's flag to match, so an imported
 *     stream continues on the kernel it would have run in the source.
 *   - a poisoned handle refuses both calls; n < 0, NULL or misaligned buffers with n > 0: MWW_EINVAL.  Frontend-only
 *     handles work (record = mask, carry, estimate). */
typedef struct mww_stream_layout {
    int64_t record_bytes;
    int32_t n_models, frontend_buffered, hop_samples;
    int32_t pending_rows[64];
    uint64_t model_hash[64];          /* hash of model k's container, its precision and state size */
    uint8_t rows_are_features[64];
} mww_stream_layout;
int mww_stream_layout_get(const mww_t *h, mww_stream_layout *out);
int mww_export_streams(mww_t *h, const int32_t *h_ids, int n, void *d_records, mww_stream_layout *out, void *cu_stream);
int mww_import_streams(mww_t *h, const int32_t *h_ids, int n, const void *d_records, const mww_stream_layout *layout,
                       void *cu_stream);

/* ---- moving resampled streams: records that carry the resampler history ----------------------------------------------
 * A stream at an input rate other than 16000 (mww_set_input_rate, mww_set_stream_rates) carries one more piece of state:
 * its resampler history.  mww_export_resampled_streams / mww_import_resampled_streams move streams with it, on any handle
 * (a plain 16 kHz one included), in either mode and across modes.
 *
 * The continuation condition.  Take a stream at rate r, L / M = 16000 / r in lowest terms, that has been given N input
 * samples.  It has emitted n0 = ceil(N L / M) outputs, and output n0 + q sits t0 + q M upsampled samples past its next
 * input, t0 = n0 M - N L = (-N L) mod M.  That output reads the inputs k - i, k = floor((t0 + q M) / L), i < H (input 0
 * being the next one): the last H inputs given and those still to come.  So every 16 kHz sample the stream emits from
 * then on depends only on its last H inputs and on t0.  As gcd(L, M) = 1, L is invertible mod M and t0 determines
 * N mod M.  A stream therefore continues bit for bit in another handle when that handle gives it the same rate and its
 * input count N' for the stream satisfies
 *     N' = N (mod M),
 * and at any other N' every later output sits at another phase of the filter.  N is the counter of mww_get_input_rate on
 * a single-rate handle, and N(t, r) = floor(t M / L) of the counter t with per-stream rates.  There the condition is the
 * same as t' = t (mod L): write t M = N L + rho with 0 <= rho < L, so t0 = (rho - t M) mod M = rho mod M.  At 8 kHz M = 1
 * and every N matches; at every other rate rho < L <= M, so t0 = rho = t M mod L, which fixes t mod L since M is
 * invertible mod L.
 *
 * At the 30 ms cadence (calls of 480 16 kHz samples) handles almost always match: t is a multiple of 480, and L = 2, 2, 1,
 * 160 and 1 at 8, 24, 32, 44.1 and 48 kHz all divide 480 (a single-rate handle's N is then a multiple of M as well).
 * Only 22.05 kHz (L = 320) can differ: t mod 320 is 0 after an even number of calls and 160 after an odd one (N mod 441 is
 * 0 or 220 on a single-rate handle, after 661 + 662 inputs per pair of calls), so two handles whose call counts differ in
 * parity are half a cycle apart.  Advancing the destination by one call fixes it.
 *
 *   - One record is the stream record of mww_export_streams, byte for byte at the same offsets, then one 496-byte part at
 *     resampler_off (== the stream layout's record_bytes): int16 hist[244], the stream's first H history samples in the
 *     handle's order (H = 52, 111, 122, 163, 222 or 243 at 8, 22.05, 24, 32, 44.1 or 48 kHz, 0 at 16000), then zeros.
 *     The resampler writes only the first H samples of a history row, and every call that sets a rate or resets a row
 *     zeroes the whole row, so the rest of a row stays zero (unless mww_set_resampler_state wrote there; the resampler
 *     never reads it).  On a 16 kHz handle the part is all zeros.
 *   - The handle's counters travel beside the records in mww_resampler_layout, and the streams' rates in h_rates_out /
 *     h_rates (int32, host memory; h_rates_out may be NULL): every check is on the host, before any device work.
 *   - Import refuses with MWW_EINVAL, before any device work and with the handle unchanged, and names the field or id: the
 *     stream layout does not fit (the fields and rules of mww_import_streams); record_bytes or resampler_off differs; a
 *     listed stream's rate in h_rates is not the destination's rate for it (or, from a single-rate handle, not the
 *     records' rate); or a listed stream fails the phase condition (the message names the rate and both phases N mod M).
 *     Ids out of range or listed twice, n < 0, NULL or misaligned buffers with n > 0 and a poisoned handle are refused as
 *     by mww_import_streams.
 *   - Import writes the listed streams' resampler history and everything mww_import_streams writes, and zeroes their audio
 *     history as it does (mww_write_audio_history comes after).  It never changes the counters or a stream's rate: set the
 *     destination's rates first with mww_set_stream_rates.
 *   - Export makes the launches of mww_export_streams plus one, import those of mww_import_streams plus one, whatever n
 *     is; n == 0 launches nothing.  Export does not change the handle. */
typedef struct mww_resampler_layout {
    int64_t record_bytes;       /* the stream record plus the resampler part */
    int64_t resampler_off;      /* == the stream layout's record_bytes */
    int32_t rate;               /* the handle's input rate, or MWW_RATE_PER_STREAM */
    int32_t reserved;
    int64_t inputs_seen;        /* the counter of mww_get_input_rate: N on a single-rate handle (t with per-stream rates) */
    int64_t samples16_seen;     /* t of mww_get_stream_rates */
} mww_resampler_layout;
/* this handle's resampled record layout and current counters, without device work */
int mww_get_resampler_layout(const mww_t *h, mww_resampler_layout *out);
int mww_export_resampled_streams(mww_t *h, const int32_t *h_ids, int n, void *d_records, mww_stream_layout *out,
                                 mww_resampler_layout *rs_out, int32_t *h_rates_out, void *cu_stream);
int mww_import_resampled_streams(mww_t *h, const int32_t *h_ids, int n, const void *d_records,
                                 const mww_stream_layout *layout, const mww_resampler_layout *rs_layout,
                                 const int32_t *h_rates, void *cu_stream);

/* ---- audio history: the last seconds of each stream's 16 kHz audio, kept on the GPU -----------------------------------
 * What a stream said around a detection (for a second-stage verifier, the pre-roll of an STT request, or false-accept audio
 * to retrain on) exists on the GPU only once G.711 decoding and resampling have run there.  A handle can keep it:
 *   - A handle has an audio history of capacity C 16 kHz samples per stream: C is 0 (off, the default) or a multiple of 8
 *     in [8, 2^22].
 *   - A stream's history is an endless run of zeros followed by every 16 kHz int16 sample the frontend consumed for that
 *     stream since the history was last zeroed: int16 audio at 16 kHz as given, float32 audio as converted (the rule of
 *     mww_features_f32), G.711 audio as decoded, and at any other input rate (one for all streams or per stream) the
 *     resampler's output.
 *   - A read of n samples (0 <= n <= C) returns the last n entries of that run for each listed stream, oldest first: the
 *     concatenation of the (decoded, resampled) input, zero-padded on the left.
 *   - Every audio entry point appends (mww_features* and mww_predict_clip*, in every form: device, _host, _remote, _multi,
 *     _f32, _g711).  mww_infer_features takes rows, not audio, and appends nothing.
 *   - Every call that zeroes a stream's window carry zeroes its history too: mww_reset (all or by id),
 *     mww_reset_device_ids and mww_reset_frontend.  mww_import_streams zeroes the history of the streams it writes (records
 *     do not carry it; their layout is unchanged; mww_write_audio_history after the import carries it).
 *     mww_set_audio_history zeroes every stream.  Nothing else touches it:
 *     not mww_set_state, mww_set_stream_rates, mww_set_model_streams or mww_set_window_step.
 *   - So after audio calls alone since the last zeroing, a stream's last frontend_buffered history samples equal
 *     carry[0, frontend_buffered) of mww_get_state whenever C >= frontend_buffered.
 *   - The history changes nothing else: features, probabilities, all state and the counters are those of a handle without
 *     it, and with C = 0 the handle issues the launches it issued before.
 *
 * mww_set_audio_history: allowed wherever a stateful call is.  Allocates a zeroed ring [n_streams][C] of int16 (ordered on
 * cu_stream) and synchronises cu_stream before it frees the old ring; C = 0 frees it.  A bad C is MWW_EINVAL, a failed
 * allocation MWW_ENOMEM; either way the old history is untouched.
 * mww_get_audio_history: the capacity, and samples_seen, the 16 kHz samples appended since the history was enabled: one
 * lockstep counter that resets do not clear, to place events on a time axis.
 * mww_read_audio_history / _device_ids: asynchronous on cu_stream, after every audio call issued before it.  Row i of d_out
 * ([n][out_stride] int16, device memory) is the last n_samples of stream ids[i]; an id listed twice is read twice.  Host
 * ids out of range are MWW_EINVAL (as mww_reset); device ids that are negative or >= n_streams give a zero row, which covers
 * the -1 slots of a detector's d_fired.  MWW_EINVAL before any device work when the handle keeps no history, n < 0,
 * n_samples is outside [0, C], out_stride < n_samples, or a buffer is NULL with work to do.  A poisoned handle refuses
 * set and read.
 * mww_write_audio_history: the inverse of the read, to carry a stream's history when it moves to another handle (read it on
 * the source, import the stream records, then write it on the destination).  After the call, stream ids[i]'s history is an
 * endless run of zeros followed by row i of d_in, n_samples long, oldest first: as if the history had been zeroed and those
 * samples appended, with samples_seen unchanged.  So sample t of the row sits at axis position samples_seen - n_samples + t,
 * in slot pos mod C of the ring, and only the last min(n_samples, C) samples can be read back.  Every other stream keeps
 * every byte.  mww_import_streams zeroes the history of the streams it writes, so write AFTER the import.  d_in is
 * [n][in_stride] int16 in memory the handle's GPU can address (peer memory from mww_ipc_open included); ids come from host
 * memory.  Asynchronous on cu_stream, one launch counted in mww_launch_count whatever n is; n == 0 launches nothing.
 * MWW_EINVAL before any device work when the handle keeps no history, n < 0, n_samples is outside [0, 2^22], in_stride <
 * n_samples, a buffer is NULL with work to do (ids with n > 0, d_in with n > 0 and n_samples > 0), or an id is out of range
 * or listed twice.  A poisoned handle refuses the call.  At 12 s of history a stream carries 384 kB: move many streams in
 * batches of ids, or carry only the samples still needed (what a verifier hears, the endpointer's lookback and the commands
 * in progress). */
int mww_set_audio_history(mww_t *h, int capacity, void *cu_stream);
int mww_get_audio_history(const mww_t *h, int *capacity, long long *samples_seen);
int mww_read_audio_history(mww_t *h, const int32_t *h_ids, int n, int n_samples, int16_t *d_out, long long out_stride, void *cu_stream);
int mww_read_audio_history_device_ids(mww_t *h, const int32_t *d_ids, int n, int n_samples, int16_t *d_out, long long out_stride,
                                      void *cu_stream);
int mww_write_audio_history(mww_t *h, const int32_t *h_ids, int n, int n_samples, const int16_t *d_in, long long in_stride,
                            void *cu_stream);

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

/* ---- Streaming detector: probabilities in, detections out, state carried across calls ---------------------------------
 * The rule the reference's ROC numbers are made with (microwakeword/test.py:337-341 and :118-135), per row and live.  A
 * detector is its own object, not part of a handle: it consumes any probability buffer [n_rows][pitch] -- what
 * mww_predict_clip*, mww_infer_features and the _multi calls write -- and no other call knows of it.
 *
 * One (window, cutoff, cooldown_slices) for all rows; per row the last window - 1 probabilities (hist, oldest first,
 * zeros after a reset), `seen` (probabilities consumed since the row's last reset) and `cooldown` (cooldown_slices after a
 * reset).  Feeding a row p[0], p[1], ... over any number of calls, split anywhere, gives what mww_false_accept_counts gives
 * on the whole sequence: with avg[i] = mean(p[i .. i + window)) in float32 (sequential sum oldest first, one division),
 * for i = 0, 1, ...: cooldown = max(cooldown - 1, 0); if cooldown == 0 and (double)avg[i] > cutoff the row fires and
 * cooldown = cooldown_slices.  A detection at i is an event with step = i + window - 1, the index since reset of the newest
 * probability of the window, and score = avg[i].  Nothing happens (no average, no cooldown tick) before a row has seen
 * `window` probabilities.  NaN never fires.  window = 1 is the plain threshold.
 *
 * Events of all rows are appended to one device buffer of `capacity` events through a device counter.  The counter keeps
 * counting past capacity: those events are dropped, per-row state advances all the same, and mww_detector_drain reports
 * the true count.  Events of one update call are in no particular order; events of different calls are in call order.
 * event.stream is the row index, or h_stream_ids[row] when the detector was created with a map (model k of a handle with
 * stream sets scores its members in list order: pass the list mww_get_model_streams returns).
 * Beside the events, d_fired [capacity] int32 holds the stream of each used event slot and -1 in every other slot, so
 * mww_reset_device_ids(h, d_fired, capacity, stream) restarts exactly the streams that fired since the last drain.
 *
 *   - create: 1 <= n_rows, 1 <= window <= 32, cooldown_slices >= 0, finite cutoff, capacity >= 1, else MWW_EINVAL; without
 *     a CUDA device MWW_ECUDA ("no CUDA device").  Messages of every detector call go to mww_last_error(NULL).
 *   - update: asynchronous on cu_stream; the first n_steps columns of each row are consumed; n_steps == 0 launches
 *     nothing; pitch >= n_steps.
 *   - drain: synchronises cu_stream, copies min(count, capacity, max_events) events to h_events (may be NULL with
 *     max_events 0), *n_events = events fired since the last drain, then clears the counter and refills d_fired with -1.
 *   - buffers: device views for callers that stay on the GPU (each out pointer may be NULL).
 *   - reset / reset_device: fresh state for all rows (NULL list) or the listed ROW indices (host / device memory; indices
 *     out of range are ignored, a row listed twice is reset once more to the same state); a constant number of launches.
 *     Events already in the buffer stay.
 *   - get_state / set_state: host buffers, synchronous (they synchronise the device), NULL pointers skipped;
 *     hist [n_rows][window - 1] oldest first, seen [n_rows], cooldown [n_rows].  set_state refuses (MWW_EINVAL) a negative
 *     seen or a cooldown outside [0, cooldown_slices]. */
typedef struct mww_detector mww_detector_t;
typedef struct mww_event { int32_t stream, reserved; int64_t step; float score; int32_t pad; } mww_event;

int mww_detector_create(int device, int n_rows, int window, double cutoff, int cooldown_slices, int capacity,
                        const int32_t *h_stream_ids, mww_detector_t **out);
int mww_detector_destroy(mww_detector_t *d);
int mww_detector_update(mww_detector_t *d, const float *d_probs, int n_steps, long long pitch, void *cu_stream);
int mww_detector_drain(mww_detector_t *d, mww_event *h_events, int max_events, long long *n_events, void *cu_stream);
int mww_detector_buffers(mww_detector_t *d, const long long **d_count, const mww_event **d_events, const int32_t **d_fired,
                         int *capacity);
int mww_detector_reset(mww_detector_t *d, const int32_t *h_rows, int n, void *cu_stream);
int mww_detector_reset_device(mww_detector_t *d, const int32_t *d_rows, int n, void *cu_stream);
int mww_detector_get_state(mww_detector_t *d, float *h_hist, long long *h_seen, int32_t *h_cooldown);
int mww_detector_set_state(mww_detector_t *d, const float *h_hist, const long long *h_seen, const int32_t *h_cooldown);

/* ---- Multi-model streaming detector: a rule per model of a handle, WAKE detections gated by a VAD model ---------------
 * A deployment that runs K wake-word and VAD models over one frontend (mww_create_multi) turns all their probabilities into
 * one event stream with one launch per call, and lets the VAD stop a wake word from firing while nobody speaks.
 *
 * The detector is created from a handle with K models.  At creation it copies each model's stride s_k and stream set S_k,
 * and it keeps them.  Each model gets a rule with one of three roles:
 *   - WAKE: (window_k, cutoff_k, cooldown_k).
 *   - VAD: (window_v, cutoff_v).  At most one model may be the VAD.
 *   - OFF: ignored.
 * At least one model must be WAKE.  Each model has one state row per member of S_k, in list order, as its probabilities do.
 * A WAKE row keeps what a plain detector row keeps: hist, seen and cooldown.  A VAD row keeps hist, seen and active, a 0/1
 * flag.
 *
 * Step timing.  An update describes one handle call.  For each model k it gives:
 *   - n_k, the steps model k ran in that call;
 *   - p_k, the model's pending rows before that call.
 * Step j of the call (0 <= j < n_k) ends at call-relative feature row e_k(j) = (j + 1) s_k - p_k - 1.  The rows that call
 * produced, R, are not passed in.  The update is accepted only if one R >= 0 fits every non-OFF model: n_k = (p_k + R) div
 * s_k and 0 <= p_k < s_k.  Otherwise it returns MWW_EINVAL before any launch.  This catches a skipped call, or a handle reset
 * that the detector was not told about, in most cases.
 *
 * Order within a stream.  A stream's steps are processed in order of e.  When a VAD step and a WAKE step end on the same
 * row, the VAD step goes first.
 *
 * VAD step.  It runs the moving average of the plain detector: float32 window_mean, a sequential sum and one division.  Then
 * active = (seen_v >= window_v) && (double)avg > cutoff_v, with seen_v counting this step.  So NaN gives false, and the flag
 * stays false until the row has seen a full window.  A stream that is not in S_v is never active.
 *
 * WAKE step (stream s = S_k[r]).  It is the plain detector's rule with one extra condition:
 *   - cooldown = max(cooldown - 1, 0);
 *   - the row fires iff cooldown == 0 && (double)avg > cutoff_k && gate, and then cooldown = cooldown_k;
 *   - gate is the active flag of stream s's VAD row, or true when no model is the VAD.
 * If the gate refuses a candidate, the row does not fire and the cooldown is not set.  Nothing happens before the row has
 * seen window_k probabilities.
 *
 * Events use the mww_event layout: stream = the global stream id; reserved = the model index k (it stays 0 for the plain
 * detector); step = model k's probability index since the row's last reset; score = the average.  d_fired holds global
 * stream ids, so mww_reset_device_ids(h, d_fired, capacity, stream) restarts every stream on which any wake word fired.
 *
 * Resets take GLOBAL stream ids.  For each listed stream it resets the stream's VAD row (zero hist, seen = 0, active = 0) and
 * every WAKE row of that stream (zero hist, seen = 0, cooldown = cooldown_k).
 *
 * Consequences: without a VAD, model k's events and state are bit-identical to those of a plain detector (n_k rows,
 * cutoff_k, window_k, cooldown_k, stream map S_k) fed the same probabilities; and events and state do not depend on how the
 * audio was split into calls, as long as every call's probabilities are passed.
 *
 *   - create: reads the handle through host-side calls only (K, strides, device, n_streams, stream sets) and does no device
 *     work on it.  MWW_EINVAL with a message for a frontend-only handle, a role outside the three, zero WAKE models or two
 *     VAD models, a window outside [1, 32], a non-finite cutoff or a negative cooldown of a used model, capacity < 1; without
 *     a CUDA device MWW_ECUDA ("no CUDA device").  The VAD's cooldown_slices is not used.
 *   - update: d_probs[k] is [n_k members][pitch[k]] in device memory (pitch[k] >= n_steps[k]); OFF models' entries,
 *     and those of models with no members or no steps, may be NULL.  One launch, or none when every n_k is 0; no
 *     host-to-device copy.  Asynchronous on cu_stream.
 *   - shared with the plain detector: mww_detector_destroy, _drain, _buffers, _reset and _reset_device (global stream ids
 *     here; a NULL list resets every stream).  mww_detector_update, _get_state and _set_state on a models detector return
 *     MWW_EINVAL, and so does mww_multi_detector_update on a plain detector.
 *   - get_state / set_state: model k's rows in list order, host buffers, synchronous, NULL pointers skipped:
 *     hist [n_k][window_k - 1] oldest first, seen [n_k], and cooldown [n_k] (WAKE) or active [n_k] (VAD).  set refuses a
 *     negative seen, a cooldown outside [0, cooldown_k] and an active outside {0, 1}; an OFF model is MWW_EINVAL. */
#define MWW_DETECT_OFF 0
#define MWW_DETECT_WAKE 1
#define MWW_DETECT_VAD 2
typedef struct mww_detect_rule { int32_t role, window, cooldown_slices, pad; double cutoff; } mww_detect_rule;
int mww_multi_detector_create(const mww_t *h, const mww_detect_rule *rules /* [K] */, int capacity, mww_detector_t **out);
int mww_multi_detector_update(mww_detector_t *d, const float *const *d_probs, const long long *pitch,
                               const int *n_steps, const int *pending_before, void *cu_stream);
int mww_multi_detector_get_state(mww_detector_t *d, int k, float *h_hist, long long *h_seen, int32_t *h_cooldown_or_active);
int mww_multi_detector_set_state(mww_detector_t *d, int k, const float *h_hist, const long long *h_seen,
                                 const int32_t *h_cooldown_or_active);

/* ---- per-row cutoffs: each stream's own sensitivity ------------------------------------------------------------------------
 * A detector starts in uniform mode: one cutoff per detector (plain) or per model (models detector), as above.  The first
 * set call with n > 0 switches it to per-row mode for good: every row keeps a cutoff c_r, all set to the create-time
 * value, and then the listed rows are written.  For a models detector that is every member row of every WAKE and VAD model.
 * The rule of a per-row detector is the rule above with (double)avg > c_r in place of (double)avg > cutoff, for WAKE firing
 * and for the VAD's active flag alike; windows, cooldowns, gating, the event layout, d_fired and step numbering do not change.
 * Consequences:
 *   1. Per-row mode with every c_r = c is bit-identical to uniform mode at c: the same set of events, and the same state.
 *   2. Row r of a per-row plain detector is bit-identical to that row of a uniform detector at c_r as long as c_r never
 *      changes; so its events are mww_false_accept_counts at c_r on everything the row was given.
 *   3. Events and state do not depend on how the probabilities were split into calls, as long as cutoff changes fall
 *      between the same steps.
 * Calls:
 *   - set: n (row, cutoff) pairs.  The plain call takes row indices; the multi call takes GLOBAL stream ids, which must be
 *     members of S_k.  Ordered on cu_stream: an update enqueued before the call uses the old cutoffs, one enqueued after it
 *     the new ones.  The host arrays may be reused as soon as the call returns.  Detector state (hist, seen, cooldown,
 *     active) is untouched, and resets keep the cutoffs.  n == 0 does nothing and does not switch mode.
 *   - MWW_EINVAL, before any device work and with the detector unchanged: a non-finite cutoff; an id out of range, listed
 *     twice or (multi) not a member of S_k; n < 0; NULL arrays with n > 0; an OFF model or a k out of range; the plain
 *     calls on a models detector and the multi calls on a plain detector.
 *   - get: every row's cutoff, host buffer [n_rows] (plain) or [n_k] in list order (multi), synchronous; the create-time
 *     value in every slot while the detector is in uniform mode.
 * The per-row kernels read 8 bytes more per row per call than the uniform ones; uniform mode runs exactly as before. */
int mww_set_detector_cutoffs(mww_detector_t *d, const int32_t *h_rows, const double *h_cutoffs, int n, void *cu_stream);
int mww_get_detector_cutoffs(mww_detector_t *d, double *h_cutoffs /* [n_rows] */);
int mww_set_multi_detector_cutoffs(mww_detector_t *d, int k, const int32_t *h_stream_ids, const double *h_cutoffs, int n,
                                   void *cu_stream);
int mww_get_multi_detector_cutoffs(mww_detector_t *d, int k, double *h_cutoffs /* [n_k], list order */);

/* ---- moving detector rows: export and import as packed records ---------------------------------------------------------
 * A server that grows, compacts or rebalances a handle moves its streams as stream records (mww_export_streams); their
 * detector rows move the same way, so that a moved stream keeps its moving average, its warm-up count, its cooldown and
 * its VAD flag.  The same calls carry the rows of every stream that stays when a new models detector replaces one after
 * mww_set_model_streams, and checkpoint some streams' rows.
 *   - Rows and ids.  A plain detector is addressed by ROW index in [0, n_rows), as mww_detector_reset is; a models detector
 *     by GLOBAL stream id in [0, n_streams) of the handle it was created from, as its reset is.  For the records a plain
 *     detector is a models detector with one WAKE model whose stream set is every row: its mask bit 0 is always set.
 *   - One record, record_bytes long (a multiple of 16), every part padded to 16 bytes:
 *         uint64  member_mask                 bit k: the stream is a member of model k and slot k holds its state
 *         for each model k whose role is not OFF, in order:
 *             float32 hist[window_k - 1]      oldest first (no bytes when window_k = 1)
 *             int64 seen; int32 flag; int32 0 flag = cooldown (WAKE) or active (VAD), as get_state reports them
 *     A plain detector of window 5 has 48-byte records.
 *   - mww_detector_layout: record_bytes, whether the detector is a models detector (multi), its model count and each
 *     model's role, window and cooldown_slices (0 for an OFF model and for the VAD).  mww_get_detector_layout fills it and
 *     does no device work; export fills it too (out may be NULL); import checks it and refuses (MWW_EINVAL) records whose
 *     layout differs from its own in multi, n_models, a model's role, a used model's window, a WAKE model's cooldown or
 *     record_bytes -- the message names the first such field.  A VAD's cooldown is not compared.
 *   - export writes one record per listed id (an id may appear twice).  For a model the stream is not a member of, the
 *     mask bit is clear and the slot is zero.  The detector does not change.
 *   - import, per used model k: a destination stream that is not a member of model k ignores slot k; a member whose
 *     record bit is set takes the slot's state; a member whose bit is clear gets fresh state, what a reset gives (zero
 *     hist, seen 0, cooldown = cooldown_k for WAKE, active 0 for VAD).  Every byte of a row that is not listed stays
 *     untouched.
 *   - What does not move: the event buffer, its counter and d_fired, which belong to the detector that produced them (drain
 *     before moving); the plain detector's stream map, because events report the destination's; the cutoffs, which are
 *     configuration the caller keeps (mww_get_detector_cutoffs / mww_set_detector_cutoffs move them).
 *   - Continuation.  A moved row that is then given the same probabilities -- for a models detector, updates with the same
 *     n_k and p_k -- produces the same events and the same state as the source row would have, bit for bit: the same
 *     model, step and score, with stream from the destination's map or id.  This holds in both kernel forms, and in uniform
 *     and per-row mode whenever the cutoffs are equal.
 *   - Both calls take host id lists and device records [n][record_bytes], 16-byte aligned, in memory the detector's GPU
 *     can address.  They are asynchronous and ordered on cu_stream, with no synchronisation: an update enqueued before an
 *     export is included in what it reads.  One launch per call whatever n is; n == 0 launches nothing and still fills /
 *     checks the layout.  The id list is staged in a buffer the detector owns (as mww_detector_reset's is), so calls on
 *     one detector from different CUDA streams must be ordered by the caller.
 *   - MWW_EINVAL before any device work, with the detector unchanged: a NULL detector or layout, n < 0, a NULL or
 *     misaligned d_records with n > 0, an id out of range, an id listed twice on import. */
typedef struct mww_detector_layout {
    int64_t record_bytes;
    int32_t multi, n_models;
    int32_t role[64], window[64], cooldown_slices[64];
} mww_detector_layout;
int mww_get_detector_layout(const mww_detector_t *d, mww_detector_layout *out);
int mww_export_detector_rows(mww_detector_t *d, const int32_t *h_ids, int n, void *d_records, mww_detector_layout *out,
                             void *cu_stream);
int mww_import_detector_rows(mww_detector_t *d, const int32_t *h_ids, int n, const void *d_records,
                             const mww_detector_layout *layout, void *cu_stream);

/* ---- second-stage verification: re-score the streams a detector fired on, with a second model, from their audio history ----
 * A small streaming model on every stream, and a larger one only on the few streams that just fired, over their last second
 * or two of audio: the usual cascade against false wakes.  A VERIFIER owns one model (any container mww_create accepts:
 * fp32 or int8 okay_nabu, any run-time geometry, hybrid), a fixed rule (n_samples, window, ignore_steps, cutoff) and `slots`
 * scratch streams.  A verify call takes a source handle `src` that keeps an audio history and n <= slots stream ids.  For
 * each index i:
 *   - id in [0, src.n_streams): a = the last n_samples entries of that stream's audio history at this point in stream order,
 *     what mww_read_audio_history returns.  p[0, m) = the probabilities a FRESH handle of the verifier's container (after
 *     create or mww_reset(NULL)) gives from one mww_predict_clip of a, with m = frames / stride and frames = (n_samples -
 *     480) / 160 + 1.  score[i] = mww_positive_scores of p with (window, ignore_steps): the max over j of the float32 mean of
 *     p[ignore_steps + j, ignore_steps + j + window), NaN when fewer than window values remain -- the positive-sample score
 *     of the reference's streaming ROC (test.py:364-373), on a fresh frontend per clip as the reference makes its positive
 *     spectrograms.  confirmed[i] = the id when (double)score[i] > cutoff, else -1; NaN never confirms.
 *   - any other id (the -1 slots of d_fired included): score[i] = NaN, confirmed[i] = -1.
 * The scores are those of that definition bit for bit, because a call runs exactly those paths: the history read kernel on
 * src, mww_reset(NULL) on the verifier's own handle, mww_predict_clip on it and mww_positive_scores.  A full reset leaves the
 * handle as create does, so a verifier reused over many calls gives what a new one gives.
 *
 * Which ids:
 *   - mww_verify_streams: d_ids [n], any int32 list in device memory (for example a plain detector's d_fired).
 *   - mww_verify_detections: a detector's event slots [0, capacity), capacity <= slots.  Slot i is events[i].stream when
 *     i < min(*d_count, capacity) and (model < 0 || events[i].reserved == model), else -1.  *d_count is read on the device,
 *     in stream order.  Events of a models detector carry global stream ids, so they are src's ids; verify each wake word
 *     with its own verifier through model = k.  Outputs are per slot: score i belongs to the drained event i, before any sort.
 *
 * Ordering and side effects:
 *   - Both calls are asynchronous on cu_stream, never synchronise the host and never allocate: every buffer, the verifier
 *     handle's clip scratch included, is sized at create.  A call issues a number of launches that depends neither on n nor
 *     on how many events fired; n == 0 in mww_verify_streams does nothing.
 *   - src and det are read, not changed: state, counters, audio history and events stay as they were.  The history read
 *     is src's own kernel on src's ring, so it counts as one launch in mww_launch_count(src), as a direct read would.
 *   - The verifier's handle is scratch, and calls on one verifier must be ordered by the caller.
 *   - The read is "now": the last n_samples when the call runs, not the samples that end at the event.  A caller that
 *     verifies at each drain, every D live calls of 480 samples, needs n_samples to cover what the verifier must hear plus
 *     D x 480 samples.  Verify BEFORE mww_reset_device_ids(src, d_fired, ...): a reset zeroes the history.
 *
 * Refusals are MWW_EINVAL with a message in mww_last_error(NULL), and leave every object unchanged.
 *   - create: slots < 1; n_samples outside [480, 2^22]; window outside [1, 32]; ignore_steps < 0; a non-finite cutoff; a
 *     rule with m < ignore_steps + window (every score would be NaN); a frontend-only (NULL) blob.  Without a CUDA device
 *     MWW_ECUDA ("no CUDA device"); a model that fails to load returns its mww_create error.
 *   - verify: a NULL verifier or src; src without an audio history or with capacity < n_samples; src, det and the verifier
 *     not on one device; n < 0 or n > slots; a detector capacity > slots; model >= K of the detector (a plain detector has
 *     K = 1); d_ids NULL with n > 0; a poisoned src.  Either output pointer may be NULL.
 *   - mww_verifier_info fills mww_verifier_desc: slots, steps (= m), device, the rule, and launches = mww_launch_count of the
 *     verifier's handle. */
typedef struct mww_verifier mww_verifier_t;
typedef struct mww_verify_rule { int32_t n_samples, window, ignore_steps, pad; double cutoff; } mww_verify_rule;
typedef struct mww_verifier_desc {
    int32_t slots, steps, device, pad;
    mww_verify_rule rule;
    int64_t launches;
} mww_verifier_desc;
int mww_verifier_create(const void *model_blob, size_t n_bytes, int device, int slots, const mww_verify_rule *rule, mww_verifier_t **out);
int mww_verifier_destroy(mww_verifier_t *v);
int mww_verifier_info(const mww_verifier_t *v, mww_verifier_desc *out);
int mww_verify_streams(mww_verifier_t *v, mww_t *src, const int32_t *d_ids, int n, float *d_scores, int32_t *d_confirmed, void *cu_stream);
int mww_verify_detections(mww_verifier_t *v, mww_t *src, mww_detector_t *det, int model, float *d_scores, int32_t *d_confirmed,
                          void *cu_stream);

/* ---- event positions: where on the audio history's axis each detection happened ---------------------------------------------
 * An event's `step` counts its row's probabilities since the row's last reset, and rows are reset from the device, so the
 * host cannot place a step in the audio.  A TIMED detector stores one more value per event: its position on the axis of the
 * audio history (mww_set_audio_history), whose sample t is the t-th 16 kHz sample appended since the history was enabled, the
 * axis samples_seen counts and the endpointer's positions use.
 *
 * Definition.  An event's position is the history-axis position of the last 16 kHz sample of the newest feature window of
 * the model step whose probability is the newest one in the firing window -- the endpointer's pos(j) of that step.
 *   - Plain detector.  An update describes its n_steps steps by a clock (last_end, step_samples): step t of the call ends at
 *     last_end - (n_steps - 1 - t) step_samples.  For an engine call, last_end = S - (buffered - (480 - hop)) - hop g and
 *     step_samples = hop stride, with S = samples_seen, buffered = frontend_buffered and g the model's pending rows, all read
 *     right after the call, as the endpointer reads them.
 *   - Models detector.  The detector copies the handle's hop at create.  An update passes row_end = S - b (b = buffered -
 *     (480 - hop), read right after the call) and each model's pending rows after the call, g_k, beside the n_k and p_k of
 *     mww_multi_detector_update.  The call produced R = n_k s_k - p_k + g_k feature rows, the same R for every non-OFF model
 *     (the step counts and p_k alone fix R only up to the strides).  WAKE step j of model k ends at
 *     row_end - hop (R - 1 - e_k(j)), with e_k(j) = (j + 1) s_k - p_k - 1, which is row_end - hop (g_k + (n_k - 1 - j) s_k):
 *     the endpointer's position formula.
 *   - Events, state, d_fired, cutoffs and records are bit for bit what an untimed detector gives from the same
 *     probabilities: the position is an extra output, not a change to the rule.
 *
 * Mode and calls (messages in mww_last_error(NULL); every refusal is MWW_EINVAL before any device work, detector unchanged):
 *   - mww_time_detector_events: makes the detector timed, for good, and allocates int64 positions[capacity], -1 in every slot.
 *     Only while its event buffer is empty: after create or a drain, with no update since; otherwise refused.  Timing a timed
 *     detector does nothing.
 *   - mww_update_detector_at / mww_update_multi_detector_at: the timed updates, one launch each as the untimed ones, which they
 *     replace: a timed detector refuses mww_detector_update and mww_multi_detector_update, an untimed one refuses these two.
 *     Refused also: step_samples < 1; NULL pending_after; pending rows after the call that give no common R; and every
 *     refusal of the untimed call.  Untimed detectors change in nothing.
 *   - mww_get_detector_positions: the device view, slot i the position of event slot i, as d_fired; -1 in unused slots (the
 *     drain refills the used ones).
 *   - mww_drain_detector_at: mww_detector_drain plus the positions of the same events into h_positions.  mww_detector_drain
 *     on a timed detector drains without them.
 *   - Orderings: update the detector right after each engine call, before the next one changes the counters; drain before
 *     mww_set_audio_history, which restarts the axis.
 *
 * Reads that end at given positions.  mww_read_audio_history_at: row i of d_out [n][out_stride] holds the n_samples samples
 * [d_ends[i] - n_samples, d_ends[i]) of stream d_ids[i], oldest first.  Entries outside [samples_seen - C, samples_seen)
 * are zeros, as are ids outside [0, n_streams): the endpointer's command-read rule.  d_ids and d_ends are in device memory,
 * so a detector's d_fired and positions go in as they are; a -1 position is an end far outside the ring.  One launch,
 * counted in mww_launch_count, no host synchronisation, and the refusals of mww_read_audio_history_device_ids plus NULL
 * d_ends with work to do.
 *
 * Verification anchored at the event.  mww_verify_detections_at, on a timed detector: slot i is verify_detections' slot id
 * plus its position P.  Its clip is [e - n_samples, e) with e = min(P + post, S), S = src's samples_seen when the call is
 * enqueued.  When the whole clip is still in the ring (e - n_samples >= S - C) the slot is scored as mww_verify_detections
 * scores it: history read, fresh verifier handle, mww_predict_clip, mww_positive_scores, confirm.  Otherwise -- an unused
 * slot, another model's event, an event whose clip has left the ring -- score NaN and confirmed -1.  An event younger than
 * post samples at verify time is heard with a shorter post-roll: its clip still has n_samples samples and ends at S.  So
 * n_samples is what the verifier hears, whatever the poll interval, and a verifier cutoff chosen offline on clips that end
 * post samples after the wake word holds in serving.  post is in [0, 2^22]; an untimed detector is refused.  The launches
 * are those of mww_verify_detections, whatever the number of events; src and det are not changed. */
int mww_time_detector_events(mww_detector_t *d);
int mww_update_detector_at(mww_detector_t *d, const float *d_probs, int n_steps, long long pitch, long long last_end, long long step_samples,
                           void *cu_stream);
int mww_update_multi_detector_at(mww_detector_t *d, const float *const *d_probs, const long long *pitch, const int *n_steps,
                                 const int *pending_before, const int *pending_after, long long row_end, void *cu_stream);
int mww_get_detector_positions(mww_detector_t *d, const int64_t **d_positions);
int mww_drain_detector_at(mww_detector_t *d, mww_event *h_events, int64_t *h_positions, int max_events, long long *n_events,
                          void *cu_stream);
int mww_read_audio_history_at(mww_t *h, const int32_t *d_ids, const long long *d_ends, int n, int n_samples, int16_t *d_out,
                              long long out_stride, void *cu_stream);
int mww_verify_detections_at(mww_verifier_t *v, mww_t *src, mww_detector_t *det, int model, long long post, float *d_scores,
                             int32_t *d_confirmed, void *cu_stream);

/* ---- grouped detection: one detection per household and window ---------------------------------------------------------------
 * A household with several satellites hears one wake word on several streams at once.  A GROUPED detector gives each row (plain
 * detector) or global stream (models detector) a group, an id in [0, n_groups) or -1 for none, and stores only the best event
 * of each group and window, so everything that reads the event buffer (d_fired, positions, anchored verification, endpointer
 * arming) does the work of one detection.  Rows of group -1 behave exactly as in the ungrouped timed detector.  A models
 * detector merges per (group, WAKE model): two wake words in one household are two answers; a VAD row never has events.
 *
 * Rule.  An update u is one mww_update_detector_at or mww_update_multi_detector_at call, taken per WAKE model k for the models
 * detector.  It has three positions on the history axis (event positions):
 *   a_u  where its first step ends: last_end - (n_steps - 1) step_samples (plain), the end of model k's step 0 (models);
 *   b_u  where its last step ends;
 *   E_u  the earliest position at which a step of any later update can end: last_end + step_samples (plain), row_end + hop
 *        (models).
 * A CANDIDATE is an event the ungrouped timed detector would store for a row of group g.  Each group (each (group, model) of a
 * models detector) is closed, or open with a deadline D_g and a best candidate.  At every update, for every group:
 *   1. If g is open and a_u >= D_g, emit its best candidate and close g.  (A models update in which model k ran no step has no
 *      a_u: step 1 is skipped, which gives what step 3 gives.)
 *   2. Take g's candidates of this update, if any: if g is open, merge them into the window; if g is closed, open it with
 *      D_g = p_min + W, p_min the smallest candidate position of this update, and merge them.  The best candidate has the
 *      highest score; ties go to the earliest position, then to the lowest stream id (then to the lowest row, where a plain
 *      detector's stream map repeats an id).  The result does not depend on thread scheduling.
 *   3. If g is open and E_u >= D_g, emit its best candidate and close g.
 * W (window_samples) is in [0, 2^22].  W = 0 is "at most one event per group per update".  Candidates of an update at or past
 * D_g still join the window when a_u < D_g: a window closes between updates, never inside one.  A clip call is one update
 * like any other; the rule is written for live calls, where a window of W samples spans about W / step_samples updates.
 *
 * Emit appends the event through the detector's own path: one slot, d_fired and its position, counted past capacity as
 * every event is.  The event keeps the winner's own stream, step, score and position, so an anchored verify hears the clip
 * around the winning detection; it is emitted up to W + step_samples after it fired, so a verify `post` of up to about W is
 * heard in full at the poll, and an endpointer armed from it must replay that far back (lookback_steps).  A grouped event also
 * records its group and `candidates`, the number of candidates merged into it; an event of a row of group -1 has group -1 and
 * candidates 1.  Per-row state (moving averages, seen, cooldowns, cutoffs) is bit for bit the ungrouped timed detector's: a
 * row that lost has still fired as far as its own cooldown is concerned.  Resets do not touch windows.
 *
 * Calls (messages in mww_last_error(NULL); refusals are MWW_EINVAL before any device work, detector unchanged):
 *   - mww_group_detector_events: makes a TIMED detector grouped, for good, every row in group -1 and every group closed.
 *     n_groups in [1, n_rows] (plain) or [1, n_streams] (models).  Refused while the detector may hold events, as
 *     mww_time_detector_events is; grouping a grouped detector is refused.
 *   - mww_set_detector_groups (rows) / mww_set_multi_detector_groups (global stream ids, one group per stream, shared by all
 *     its WAKE models): the listed ids' groups, ordered on cu_stream.  Ids out of range or listed twice, and groups outside
 *     [-1, n_groups), are refused.  Groups may change between any two calls; an open window keeps its candidates.
 *     mww_get_detector_groups / mww_get_multi_detector_groups: every row's or stream's group.
 *   - The timed updates run the grouped kernels on a grouped detector: two launches (the update, then the close of every
 *     group), whatever the number of events.  Ungrouped and untimed detectors run exactly the kernels they ran before.
 *   - mww_flush_detector_groups: emits every open window now (one launch).
 *   - mww_drain_detector_groups: mww_drain_detector_at plus each event's group and candidates.
 *   - mww_get_detector_group_windows / mww_set_detector_group_windows: every group slot's window, n_groups x n_wake entries
 *     (n_wake 1 for a plain detector, its WAKE models for a models detector): slot g n_wake + w, w the index of the WAKE model
 *     among the WAKE models in model order.  Both wait for the device.  Set refuses open not in {0, 1} and an open window with
 *     candidates < 1.  With the groups, they are a grouped detector's checkpoint.
 *   - Moves: detector records carry no windows and no groups (a destination keeps its own groups); export_rows and
 *     import_rows leave the windows alone.  Drain before a move as always, and flush the source too, or accept that its open
 *     windows are lost for the streams that leave. */
typedef struct {
    int64_t deadline;         /* D_g, when open */
    int64_t sample, step;     /* the best candidate's position and step */
    int32_t stream;           /* its stream (global stream id for a models detector) */
    float score;              /* its score */
    int32_t candidates;       /* candidates merged into the window */
    int32_t open;             /* 1: open, 0: closed */
} mww_group_window;
int mww_group_detector_events(mww_detector_t *d, int n_groups, long long window_samples);
int mww_set_detector_groups(mww_detector_t *d, const int32_t *h_rows, const int32_t *h_groups, int n, void *cu_stream);
int mww_get_detector_groups(mww_detector_t *d, int32_t *h_groups);
int mww_set_multi_detector_groups(mww_detector_t *d, const int32_t *h_stream_ids, const int32_t *h_groups, int n, void *cu_stream);
int mww_get_multi_detector_groups(mww_detector_t *d, int32_t *h_groups);
int mww_flush_detector_groups(mww_detector_t *d, void *cu_stream);
int mww_drain_detector_groups(mww_detector_t *d, mww_event *h_events, int64_t *h_positions, int32_t *h_groups, int32_t *h_candidates,
                              int max_events, long long *n_events, void *cu_stream);
int mww_get_detector_group_windows(mww_detector_t *d, mww_group_window *h_windows);
int mww_set_detector_group_windows(mww_detector_t *d, const mww_group_window *h_windows);

/* ---- group arbitration: the satellite that heard the wake word best answers ----------------------------------------------------
 * Grouped detection picks a window's winner by score.  Every satellite that hears the word clearly saturates an int8 model's
 * score (multiples of 1/256), and all streams of a handle step in lockstep, so the score and position tie and the lowest stream
 * id answers.  An ARBITRATED detector picks the candidate that heard the word loudest over its own background instead: the
 * device next to the speaker, not the one across the room.  It is opt-in; a detector that is not arbitrated is unchanged.
 *
 * Rule.  A grouped, timed detector is bound to a handle src with (speech_samples Ls, noise_samples Ln), both in [480, 2^20],
 * Ls + Ln at most src's history capacity.  For a candidate (grouped detection) of stream s at position P:
 *   - Spans: speech [P - Ls, P), noise [P - Ls - Ln, P - Ls), read from src's history ring with the read-at rule: a position
 *     outside [S - C, S) reads as zero, S src's samples_seen at the update (the update runs right after the engine call).
 *   - Energy of a span of L int16 samples x: q = (double)sum x^2 (exact: below 2^53 for L <= 2^22), r = (double)sum x,
 *     e = (q - r r / L) / L, every operation a separately rounded IEEE double operation (no fused multiply-add): the
 *     mean-removed power, so that a microphone's DC offset does not make a satellite look loud.
 *   - level = (float)((e_speech + 1) / (e_noise + 1)), rounded to nearest.  The + 1 is a floor of one LSB^2, so an all-zero
 *     (noise-gated) span divides by 1.  10 log10(level) is the level in dB.
 *   - Order: the best candidate of a group and window has the highest level, then the highest score, then the earliest
 *     position, then the lowest row (plain detector) or lowest global stream (models detector).  Steps 1 to 3 of grouped
 *     detection are unchanged; when an update's best joins an open window, "better" is this order and an exact tie keeps the
 *     earlier candidate.
 *   - Per-row state is bit for bit the ungrouped timed detector's, and rows of group -1 store their events as before.  Each
 *     emitted winner carries its level; an event of a row of group -1 carries NaN.
 * What the level cannot know: how far each device's microphone gain, enclosure and placement differ; a satellite with a hotter
 * microphone looks closer.  The level compares each device with its own background, which cancels a fixed gain only where
 * both spans see it alike.
 *
 * Calls (messages in mww_last_error(NULL); refusals are MWW_EINVAL before any device work, detector unchanged):
 *   - mww_arbitrate_detector_groups: makes a grouped detector arbitrated, for good, every window level 0.  Refused when the
 *     detector is not grouped, is already arbitrated or may hold events; when src is NULL, poisoned or on another device;
 *     when a row's stream (plain: its stream_ids entry or row; models: every global stream) is outside src; when Ls or Ln is
 *     out of range or Ls + Ln exceeds src's history capacity.  src must outlive the detector.
 *   - The timed updates and mww_flush_detector_groups then run the arbitrated kernels: the same two launches per update (one
 *     per flush) whatever the number of events.  An update is refused while src's history holds fewer than Ls + Ln samples
 *     (mww_set_audio_history), lacks a stream a row reads, or is poisoned.
 *   - mww_drain_detector_arbitrated: mww_drain_detector_groups plus each event's level.
 *   - mww_get_detector_group_levels / mww_set_detector_group_levels: every group slot's window level (slots as the windows'),
 *     part of the checkpoint with the windows and groups.  Both wait for the device; set refuses a level that is NaN,
 *     infinite or negative.  Detector records carry no levels, as they carry no windows. */
int mww_arbitrate_detector_groups(mww_detector_t *d, mww_t *src, int speech_samples, int noise_samples);
int mww_drain_detector_arbitrated(mww_detector_t *d, mww_event *h_events, int64_t *h_positions, int32_t *h_groups, int32_t *h_candidates,
                                  float *h_levels, int max_events, long long *n_events, void *cu_stream);
int mww_get_detector_group_levels(mww_detector_t *d, float *h_levels);
int mww_set_detector_group_levels(mww_detector_t *d, const float *h_levels);

/* ---- media guard: suppress the detections that many households, or a registered media clip, heard alike ---------------------
 * A TV advert, a podcast or a broadcast that says the wake word makes thousands of households fire within a second, and every
 * one of those detections is a true positive for the wake model and the verifier.  A broadcast is the same audio heard in many
 * homes at once; a MEDIA GUARD fingerprints each detection's clip and takes the ones that match other households' recent
 * detections, or a registered media clip, out of what gets armed.  Like a verifier it works on slots.  Slot i has a stream id,
 * an end position e_i, a position P_i on the history axis (event positions) and a household h_i.
 *
 * Clip.  The n_samples 16 kHz samples [e_i - n_samples, e_i) of that stream's audio history, what mww_read_audio_history_at
 * returns.  A slot is INVALID when its id is -1 or outside [0, src.n_streams), when it holds another model's event, or when its
 * clip has partly left the ring: e_i - n_samples < S - C (S = src's samples_seen when the call is enqueued, C its capacity).
 *   - mww_media_check_streams: d_ids[i], e_i = P_i = d_ends[i], h_i = d_households[i] (-1 for every slot when d_households is
 *     NULL).
 *   - mww_media_check_detections_at: event slot i of a timed detector, as mww_verify_detections_at takes it: the event's stream,
 *     P_i its position, e_i = min(P_i + post, S); h_i the event's group on a grouped detector, -1 on an ungrouped one (so every
 *     stream is its own household).
 * Features.  F = the rows a fresh frontend (the guard's own frontend-only handle after mww_reset(NULL)) emits from one
 * mww_features call over the clip: T = (n_samples - 480) / 160 + 1 rows of 40 uint16 values, the verifier's fresh frontend
 * per clip.
 * Fingerprint.  One uint64 word per frame t in [1, T): bit c, c in [0, 39), is set when the int32 value
 *     (F[t][c] - F[t][c+1]) - (F[t-1][c] - F[t-1][c+1]) > 0
 * (the Haitsma-Kalker energy-difference sign); bits 39..63 are zero.  A clip has W = T - 1 words.
 * Distance.  For fingerprints x (n_x words) and y (n_y words) at lag l, the overlap O(l) = #{t : 0 <= t < n_x, 0 <= t + l < n_y}
 * and the mismatches m(l) = sum over it of popcount(x[t] XOR y[t + l]).  x and y MATCH when some allowed l has O(l) >=
 * min_overlap and m(l) 1000 <= max_ber_milli 39 O(l): integers, so the result is exact.  Between two detections the allowed
 * lags are |l| <= max_lag frames (the jitter between where different households' detectors fire on the same content);
 * against a registered clip every l with O(l) >= min_overlap is allowed, so the clip may sit anywhere in a long advert.
 * Rule of one check call.  For each valid slot i:
 *   - matches[i] = the number of candidates j that are (1) one of this call's other valid slots or one of the ring's entries,
 *     (2) in another household -- two events are in one household when h_i == h_j >= 0, or h_i == h_j == -1 on one stream --,
 *     (3) within |P_j - P_i| <= window_samples, and (4) match i;
 *   - media[i] = bit 0 when i matches any registered clip | bit 1 when matches[i] >= min_matches;
 *   - passed[i] = -1 when media[i] != 0, else d_confirmed[i], or the slot's stream id when d_confirmed is NULL: it goes
 *     straight into mww_endpointer_arm_device.
 * An invalid slot gives matches -1, media 0, and passed its confirmed id: the guard never blocks what it cannot hear.  A slot's
 * stream id is d_ids[i], or the event's stream (-1 for an unused slot or another model's event).
 * Ring.  After matching, every valid slot is appended to a ring of `ring` entries in slot order, flagged or not: its
 * fingerprint, stream, household and P.  When the ring is full the oldest entry is overwritten.  So a detection is matched
 * against the ones of earlier checks within the window, however the polls cut the wave.
 *
 * Rule fields (mww_media_rule; fixed at create):  n_samples in [640, 160000]; max_lag in [0, 64]; min_overlap in [1, W] with
 * max_lag <= W - min_overlap; max_ber_milli in [0, 500]; min_matches >= 1; ring in [0, 2^20]; window_samples in [0, 2^40];
 * max_media (registered clips) in [0, 4096]; max_media_samples in [0, 2^24], and when max_media > 0 at least 640 and with
 * (max_media_samples - 480) / 160 >= min_overlap; max_media times that word count at most 2^27.
 *
 * Calls (refusals are MWW_EINVAL with a message in mww_last_error(NULL), before any device work, every object unchanged):
 *   - mww_media_guard_create: slots >= 1 and the rule above; MWW_ECUDA without a device.  _destroy waits for the device.
 *     mww_media_guard_info fills mww_media_guard_desc: slots, frames (T), device, n_media (registered clips), the rule,
 *     ring_count (slots appended since the last clear), ring_fill = min(ring_count, ring), and launches: the kernel launches
 *     of the guard and its frontend handles since create.  It waits for the device.
 *   - mww_media_check_streams / mww_media_check_detections_at: outputs [n] (capacity for a detector), each may be NULL;
 *     d_confirmed [n] may be NULL.  Refused: a NULL guard or src; src without an audio history or with capacity < n_samples; src,
 *     det and the guard not on one device; n < 0 or n > slots; a detector capacity > slots; d_ids or d_ends NULL with n > 0;
 *     a poisoned src; an untimed detector; model >= the detector's model count (model < 0: every model; model = k: one wake word
 *     of a models detector); post outside [0, 2^22].  n == 0 does nothing.
 *   - Ordering and side effects, as for the verifier: asynchronous on cu_stream, no host synchronisation and no allocation after
 *     create; src and det are read, not changed (the history read is src's own kernel, one launch of mww_launch_count(src));
 *     check BEFORE mww_reset_device_ids(src, ...), which zeroes the history.  A call launches the same kernels whatever n and
 *     however many events fired.  Calls on one guard are ordered by the caller on one stream.
 *   - mww_media_register: fingerprints n_samples 16 kHz int16 samples in device memory through the same frontend path (a fresh
 *     frontend, W_k = (n_samples - 480) / 160 words) and appends them as registered clip *index.  Refused: a NULL guard or audio,
 *     a full list, n_samples above max_media_samples or with W_k < min_overlap.  Asynchronous on cu_stream.
 *     mww_media_clear_registered empties the list.
 *   - mww_media_clear_ring empties the ring; use it after mww_set_audio_history, which restarts the axis.  It waits for the
 *     device.
 *   - mww_media_get_state / mww_media_set_state: the ring and the registered clips as one host blob, for checkpoints.  Get with
 *     h_state NULL writes the blob's size to *n_bytes; otherwise *n_bytes must be at least that size.  Both wait for the device.
 *     Layout: int64 ring_count; int32 words (W), ring, n_media, pad; int64 media_words; then uint64 ring_fp[ring][W], int64
 *     ring_pos[ring], int32 ring_stream[ring], int32 ring_household[ring]; then int64 clip_words[n_media] and the uint64
 *     words of every clip, in order.  Set refuses a blob of another size, W or ring, more clips than max_media, a clip length
 *     outside [min_overlap, the longest registrable] or a sum that is not media_words. */
typedef struct mww_media_guard mww_media_guard_t;
typedef struct mww_media_rule {
    int32_t n_samples, max_lag, min_overlap, max_ber_milli;
    int32_t min_matches, ring, max_media, max_media_samples;
    int64_t window_samples;
} mww_media_rule;
typedef struct mww_media_guard_desc {
    int32_t slots, frames, device, n_media;
    mww_media_rule rule;
    int64_t ring_fill, ring_count, launches;
} mww_media_guard_desc;
int mww_media_guard_create(int device, int slots, const mww_media_rule *rule, mww_media_guard_t **out);
int mww_media_guard_destroy(mww_media_guard_t *g);
int mww_media_guard_info(const mww_media_guard_t *g, mww_media_guard_desc *out);
int mww_media_check_streams(mww_media_guard_t *g, mww_t *src, const int32_t *d_ids, const long long *d_ends, const int32_t *d_households, int n,
                            const int32_t *d_confirmed, int32_t *d_matches, int32_t *d_media, int32_t *d_passed, void *cu_stream);
int mww_media_check_detections_at(mww_media_guard_t *g, mww_t *src, mww_detector_t *det, int model, long long post, const int32_t *d_confirmed,
                                  int32_t *d_matches, int32_t *d_media, int32_t *d_passed, void *cu_stream);
int mww_media_register(mww_media_guard_t *g, const int16_t *d_audio, int n_samples, int *index, void *cu_stream);
int mww_media_clear_registered(mww_media_guard_t *g);
int mww_media_clear_ring(mww_media_guard_t *g);
int mww_media_get_state(mww_media_guard_t *g, void *h_state, long long *n_bytes);
int mww_media_set_state(mww_media_guard_t *g, const void *h_state, long long n_bytes);

/* ---- playback guard: suppress the detections a device's own playback said ---------------------------------------------------
 * A satellite plays what the server sends it -- replies, music -- and its microphone hears that playback.  A reply that says
 * the wake word, or a word close to it, fires the stream, and for the wake model and the verifier that is a true positive.
 * The server knows what it sent to each stream, so a PLAYBACK GUARD keeps that playback on the GPU and asks, at each detection:
 * did the device itself say the wake word in the delay window before it?  A wake model answers that on the clean playback.
 *
 * Binding and axis.  A guard is bound at create to a handle h that keeps an audio history, as an endpointer is, and uses h's
 * history axis: position t is the t-th 16 kHz sample appended since the history was enabled (samples_seen).  The guard reads
 * h's counters on the host only and never launches work on h.
 * Playback.  For each stream s, pb_s maps axis positions to int16, 0 everywhere until written.
 * Rows.  The guard owns `rows` ring rows of C int16 samples (C a multiple of 8 in [8, 2^22]).  A stream that is playing holds
 * one row with a head w, the end of its latest write; the row holds positions [w - C, w).  Reading position p gives pb_s(p)
 * when w - C <= p < w, else 0; a stream without a row reads 0 everywhere.
 * Write (s, a, x[0, n)).  If s has no row it takes the lowest-numbered free row (ids in list order), which counts as holding
 * zeros with head a - C.  Then, with w' = max(w, a + n): positions [max(a, w' - C), a + n) get x; when a > w the gap
 * [max(w, w' - C), a) gets zeros; every other held position keeps its value; the head becomes w'.  So a write into the past
 * (a + n <= w) overwrites only what the ring still holds, and writes ahead of samples_seen are allowed.
 * Release.  At the start of every write call every row whose head w <= S - C is freed (S = h's samples_seen at the call).  No
 * check can see it: a heard clip starts at r0 >= S - C, and everything such a row holds lies before w <= S - C.  A write that
 * needs more rows than are free after the release is refused with MWW_ENOMEM, and nothing is written or freed.  Reset(ids)
 * frees those streams' rows; a whole reset (NULL) frees every row -- use it after mww_set_audio_history, which restarts the axis.
 * Slots.  As the verifier's: slot i has a stream id and a clip end e_i.
 *   - mww_playback_check_streams: d_ids[i] and d_ends[i].
 *   - mww_playback_check_detections_at: event slot i of a timed detector under mww_verify_detections_at's slot rule: the event's
 *     stream (-1 for an unused slot or another model's event), its position P, e_i = min(P + post, S); model < 0: every model,
 *     k: one wake word of a models detector.
 * Reference clip.  L_ref = n_samples + max_delay - min_delay.  Slot i's reference clip is pb_s over [r0, r1), r1 = e_i -
 * min_delay, r0 = r1 - L_ref: the union of the playback windows [e - n_samples - d, e - d) of every delay d in [min_delay,
 * max_delay], d being the samples between a playback position and where the microphone hears it.
 * Heard.  A slot is heard when its id is in [0, n_streams), the stream holds a row, r0 >= S - C, r0 >= w - C and r0 < w: the row
 * still holds the whole window, and the window starts before the head, so some of it has been written.
 * Score and decision.  For a heard slot, score = exactly what a verifier of the guard's container with rule (L_ref, window,
 * ignore_steps, cutoff) gives on the reference clip (a fresh handle, one mww_predict_clip, mww_positive_scores with (window,
 * ignore_steps)); flagged = (double)score > cutoff, which NaN never is; passed = -1 when flagged, else d_confirmed[i], or the
 * slot's stream id when d_confirmed is NULL.  An unheard slot gets score NaN, flagged 0 and passed its confirmed id: the guard
 * never blocks what it cannot hear.  passed goes straight into mww_endpointer_arm_device, after the media guard's passed.
 * What it cannot know:
 *   - The rule never looks at the microphone audio.  A detection is suppressed because the device itself said something the
 *     model scores above cutoff in the delay window.  So a user who says the wake word over music passes, and one who says it
 *     over the device saying it is suppressed.
 *   - Playback that fires the detector only after the room has coloured it is missed; a guard cutoff below the detector's
 *     widens the net.
 *   - C must cover the longest write made ahead of time plus L_ref.  Real-time writes need only L_ref plus the poll latency.
 *
 * Calls (refusals are MWW_EINVAL with a message in mww_last_error(NULL), before any device work, the guard unchanged; the one
 * other code is MWW_ENOMEM for a write that runs out of rows):
 *   - mww_playback_guard_create: refused for a handle without an audio history or frontend-only; a NULL blob; slots < 1; rows
 *     outside [1, n_streams]; a bad capacity C; n_samples < 480; delays outside 0 <= min_delay <= max_delay <= 2^22; L_ref >
 *     min(C, 2^22); and the verifier's refusals of window, ignore_steps and cutoff, "every score would be NaN" included.
 *     MWW_ECUDA without a device.  _destroy waits for the device.  mww_playback_guard_info fills mww_playback_guard_desc: slots,
 *     steps (the verifier's m), rows, rows_used, capacity (C), l_ref, device, the rule and launches (the guard's kernel launches
 *     and its verifier handle's).
 *   - mww_playback_write: n distinct ids in [0, n_streams) with starts in [-2^50, 2^50] (host memory), each writing row i of
 *     d_audio [n][audio_stride] (n_samples in [0, 2^22], audio_stride >= n_samples).  One host-to-device copy of the call's
 *     (row, start, old head) list and one launch, whatever n.
 *   - mww_playback_read: d_out [n][out_stride] row i = pb of stream d_ids[i] over [d_ends[i] - n_samples, d_ends[i]) by the read
 *     rule (0 for an id outside [0, n_streams)); ids and ends in device memory.
 *   - mww_playback_reset: frees the rows of the n listed ids (host memory), or of every stream when h_ids is NULL.
 *   - mww_playback_get_heads: h_rows [n_streams] (-1: no row) and h_heads [n_streams] (0 without a row), either may be NULL;
 *     the host's copy, so it needs no device synchronisation.  With mww_playback_read and mww_playback_write it moves a stream's
 *     playback to another guard.
 *   - mww_playback_check_streams / mww_playback_check_detections_at: outputs [n] (capacity for a detector), each may be NULL;
 *     d_confirmed may be NULL.  Refused as the verifier's checks are, with the bound handle in place of src: a NULL guard; the
 *     bound handle without an audio history, or poisoned; n < 0 or n > slots; d_ids or d_ends NULL with n > 0; a detector
 *     capacity > slots or on another device; model >= the detector's model count; an untimed detector; post outside [0, 2^22].
 *     A check makes a constant number of launches whatever the number of events: the slots and reference read, the model's
 *     reset and clip, the positive scores, the decision.  n == 0 does nothing.
 *   - Nothing allocates after create; every call is asynchronous on cu_stream, and calls on one guard are ordered by the caller. */
typedef struct mww_playback_guard mww_playback_guard_t;
typedef struct mww_playback_rule { int32_t n_samples, window, ignore_steps, pad; int64_t min_delay, max_delay; double cutoff; } mww_playback_rule;
typedef struct mww_playback_guard_desc {
    int32_t slots, steps, rows, rows_used;
    int32_t capacity, l_ref, device, pad;
    mww_playback_rule rule;
    int64_t launches;
} mww_playback_guard_desc;
int mww_playback_guard_create(const mww_t *h, const void *model_blob, size_t n_bytes, int slots, int rows, int capacity,
                              const mww_playback_rule *rule, mww_playback_guard_t **out);
int mww_playback_guard_destroy(mww_playback_guard_t *g);
int mww_playback_guard_info(const mww_playback_guard_t *g, mww_playback_guard_desc *out);
int mww_playback_write(mww_playback_guard_t *g, const int32_t *h_ids, const long long *h_starts, int n,
                       const int16_t *d_audio, int n_samples, long long audio_stride, void *cu_stream);
int mww_playback_read(mww_playback_guard_t *g, const int32_t *d_ids, const long long *d_ends, int n, int n_samples,
                      int16_t *d_out, long long out_stride, void *cu_stream);
int mww_playback_reset(mww_playback_guard_t *g, const int32_t *h_ids, int n, void *cu_stream);
int mww_playback_get_heads(const mww_playback_guard_t *g, int32_t *h_rows, int64_t *h_heads);
int mww_playback_check_streams(mww_playback_guard_t *g, const int32_t *d_ids, const long long *d_ends, int n, const int32_t *d_confirmed,
                               float *d_scores, int32_t *d_flagged, int32_t *d_passed, void *cu_stream);
int mww_playback_check_detections_at(mww_playback_guard_t *g, mww_detector_t *det, int model, long long post, const int32_t *d_confirmed,
                                     float *d_scores, int32_t *d_flagged, int32_t *d_passed, void *cu_stream);

/* ---- endpointing: where the spoken command after a wake word ends, and its clip from the audio history ----------------------
 * After a wake word a voice assistant sends the command that follows to speech-to-text and stops when the speaker stops.  An
 * ENDPOINTER finds that end on the GPU, per stream, from a VAD model's probabilities, and cuts each command's clip from the
 * audio history, with no host round trip.
 *
 * What it is bound to.  An endpointer is created from a handle h that keeps an audio history and a model index k, whose
 * probabilities it reads as speech probabilities (any model works).  At create it copies, host side only, the model's
 * stride s, its stream set S_k (all streams when it has none) and hop_samples.  Each member of S_k has one row, in list
 * order, as the model's probabilities do (the VAD role of a models detector follows the same convention).
 *
 * Time axis.  Every position is on the audio history's axis (samples_seen of mww_get_audio_history), so a position reads
 * back from the ring directly.  An update describes the handle call made just before it.  Right after that call the
 * endpointer reads h's host-side counters: S = samples_seen, b = frontend_buffered - (480 - hop) and g = model k's pending
 * rows.  The call's n steps end at
 *     pos(j) = S - b - hop (g + (n - 1 - j) s),   j = 0 .. n - 1,
 * the last 16 kHz sample of the newest feature window of step j.  Derivation: the frontend emits a row when it holds 480
 * samples and then drops hop of them, so a call of n16 samples that emits R rows leaves buffered' = buffered + n16 - R hop,
 * and after any row the carry holds the last 480 - hop samples of the newest window plus the b samples that came after it:
 * buffered = (480 - hop) + b, so the newest row's window ends at S - b (before the first row, b < 0 and S - b is where a row
 * before it would have ended, one hop before the first).  Model k runs a step on every s rows and holds the g newest, so
 * its newest step ends g rows, hop g samples, before the newest row, and each earlier step s rows before the next.  In
 * 480-sample live calls b = 0.  The endpointer keeps the counters of the previous update (S', b', g'); the rows emitted
 * since then are R = ((S - b) - (S' - b')) / hop, and an update is refused (MWW_EINVAL, before any launch) unless R is a
 * whole number >= 0 and n s = g' + R - g, as the models detector refuses inconsistent updates: this catches a skipped
 * update.  After a full reset of the handle (mww_reset(NULL), mww_reset_frontend) or mww_set_audio_history, reset the whole
 * endpointer, which takes the handle's counters as its new baseline.
 *
 * Speech flag.  Every member row runs the VAD rule of the models detector on every step, armed or not: float32 window_mean
 * over vad_window (1 .. 32) probabilities, and speech = seen >= vad_window && (double)avg > vad_cutoff, with seen counting
 * this step.  So a row's flag is the `active` flag of a models detector's VAD row with the same window and cutoff, fed the
 * same probabilities, bit for bit.  Each row keeps its last 64 flags in a uint64 (bit i: i steps before the newest); a flag
 * from before a reset, or from before the row had a full window, is 0.
 *
 * Segmenter.  It runs on armed rows only.  State: elapsed, run, silence, heard, start_sample, speech_end_sample.  For each
 * step in order, with flag f at position p (the first step after arming sets start_sample = speech_end_sample = p - s hop):
 *     elapsed += 1
 *     if f:  run += 1; silence = 0; if run >= speech_steps: heard = 1;  if heard: speech_end_sample = p
 *     else:  run = 0;  silence += 1
 *     end with END_OF_SPEECH if heard && silence >= silence_steps
 *     else NO_SPEECH         if !heard && elapsed >= timeout_steps
 *     else MAX_LENGTH        if elapsed >= max_steps
 * A row that ends emits one event and disarms; a row that is not armed holds zero segmenter state.
 *
 * Arming.  arm(ids) takes GLOBAL stream ids from the host (ids outside [0, n_streams) are MWW_EINVAL) or the device (ids
 * outside the set and -1 are ignored, so a verifier's d_confirmed or a detector's d_fired is passed in directly).  A host id
 * in range that is not a member of S_k is ignored, and an id listed twice arms once.  Arming a row gives it fresh segmenter
 * state (re-arming an armed row restarts it), then replays its last L = min(lookback_steps, steps consumed since create or
 * the last whole reset) flags, oldest first, at their recorded positions (lookback_steps in 0 .. 64).  So arming with
 * lookback L is the same as having armed L steps earlier, which covers the detector -> verifier -> arm latency: a drain
 * every 33 live calls is about 1 s, and 64 steps are 1.92 s at stride 3.  A replay that reaches an end condition emits its
 * event during the arm call.  A replay that reaches back over the wake word hears it as speech: the segment then starts
 * before the wake word, and a pause of silence_steps after it ends the command with END_OF_SPEECH before the command is
 * spoken.  Choose lookback_steps (the latency to cover) and silence_steps (longer than the pause a speaker makes after the
 * wake word) together, or arm at the detection's position instead ("positioned arm" below).  disarm(ids) cancels without an event.  reset(ids) gives those rows fresh VAD and segmenter state:
 * call it when the handle's streams are reset.  A whole reset (ids NULL) does that for every row, takes the handle's
 * counters as the new baseline and forgets the steps consumed and their positions, so no replay reaches across it (the
 * axis may have restarted: mww_set_audio_history sets samples_seen back to 0).
 *
 * Outputs, as the detectors keep them:
 *   - events through a device counter into `capacity` slots; the count keeps going past capacity, and drain reports the
 *     true count.  end_sample is the position of the ending step; speech_end_sample is start_sample if speech was never
 *     heard; steps is elapsed at the end.
 *   - d_ended [capacity]: the stream of each used slot, -1 elsewhere.  It feeds mww_reset_device_ids and
 *     mww_read_audio_history_device_ids.
 *   - d_armed [n_rows]: the global id of every armed row, -1 elsewhere.  With the history read it lets a server stream the
 *     new audio of commands in progress to a streaming STT at each poll.
 *   - drain synchronises cu_stream, copies min(count, capacity, max_events) events to h_events, *n_events = the events since
 *     the last drain, then clears the counter and refills d_ended with -1.
 *
 * Command read.  mww_endpointer_read_commands writes, for each used event slot i, samples [a, e) of the stream's history,
 * oldest first, into row i of d_out [capacity][out_stride] int16: a = start_sample - pre, e = min(speech_end_sample + post,
 * end_sample) for END_OF_SPEECH and end_sample otherwise, the length capped at max_samples keeping the beginning.  Entries
 * outside the ring are zeros: those older than samples_seen - C and those from before a reset, as the history rule already
 * defines them, and those at or after samples_seen.  d_lengths[i] (int32) is the length, 0 for unused slots; row entries
 * past the length are zeros.  The event count is read on the device.  One launch, no host synchronisation; read BEFORE the
 * drain, and BEFORE any reset of those streams: a reset zeroes their history.
 *
 * Calls.  Update, arm, disarm, reset and read are asynchronous on cu_stream, never allocate and issue one launch each,
 * whatever n is and however many rows are armed or ended; a host id list is copied into a buffer the endpointer owns, so
 * calls on one endpointer from different CUDA streams must be ordered by the caller.  None of them launches work on h, and
 * mww_endpointer_info reports the endpointer's own launches.  Events and state do not depend on how the audio was split into
 * calls, as long as every call's probabilities are passed.
 *   - update: d_probs [n_rows][pitch] (pitch >= n), the model's probabilities of the call just made on h.
 *   - get_state / set_state: host buffers, synchronous, NULL pointers skipped; per row hist [n_rows][vad_window - 1] oldest
 *     first, seen, flags, armed, elapsed, run, silence, heard, start_sample, speech_end_sample; and the endpointer's
 *     baseline (samples_seen, buffered, pending), steps consumed since create or the last whole reset and positions[i], the position of the step i
 *     steps before the newest (0 where there is none).  set refuses a negative seen or count, heard outside {0, 1}, an armed
 *     value that is neither -1 nor the row's stream, and a baseline outside the handle's ranges.
 *
 * Refusals are MWW_EINVAL with a message in mww_last_error(NULL), before any device work.
 *   - create: a handle without history; a frontend-only handle or k out of range; vad_window outside [1, 32] or a
 *     non-finite vad_cutoff; speech_steps, silence_steps, timeout_steps or max_steps below 1; lookback_steps outside
 *     [0, 64]; capacity < 1.  Without a CUDA device MWW_ECUDA ("no CUDA device").
 *   - update: n < 0, pitch < n, NULL probabilities with n > 0, and the consistency check above.
 *   - read: a different handle than the endpointer's, pre < 0, post < 0, max_samples outside [0, 2^22], out_stride <
 *     max_samples, NULL buffers, or a handle that no longer keeps a history. */
#define MWW_ENDPOINT_END_OF_SPEECH 1
#define MWW_ENDPOINT_NO_SPEECH 2
#define MWW_ENDPOINT_MAX_LENGTH 3
typedef struct mww_endpointer mww_endpointer_t;
typedef struct mww_endpoint_rule {
    int32_t vad_window, speech_steps, silence_steps, timeout_steps, max_steps, lookback_steps;
    double vad_cutoff;
} mww_endpoint_rule;
typedef struct mww_endpoint_event {
    int32_t stream, reason;
    int64_t start_sample, end_sample, speech_end_sample;
    int32_t steps, pad;
} mww_endpoint_event;
typedef struct mww_endpointer_desc {
    int32_t n_rows, model, stride, hop_samples, capacity, device;
    mww_endpoint_rule rule;
    int64_t steps, launches;
} mww_endpointer_desc;
typedef struct mww_endpoint_state {
    float *hist;
    int64_t *seen;
    uint64_t *flags;
    int32_t *armed, *elapsed, *run, *silence, *heard;
    int64_t *start_sample, *speech_end_sample;
    int64_t samples_seen, buffered, pending, steps;
    int64_t positions[64];
} mww_endpoint_state;
int mww_endpointer_create(const mww_t *h, int model, const mww_endpoint_rule *rule, int capacity, mww_endpointer_t **out);
int mww_endpointer_destroy(mww_endpointer_t *ep);
int mww_endpointer_info(const mww_endpointer_t *ep, mww_endpointer_desc *out);
int mww_endpointer_update(mww_endpointer_t *ep, const float *d_probs, int n, long long pitch, void *cu_stream);
int mww_endpointer_arm(mww_endpointer_t *ep, const int32_t *h_ids, int n, void *cu_stream);
int mww_endpointer_arm_device(mww_endpointer_t *ep, const int32_t *d_ids, int n, void *cu_stream);
int mww_endpointer_disarm(mww_endpointer_t *ep, const int32_t *h_ids, int n, void *cu_stream);
int mww_endpointer_reset(mww_endpointer_t *ep, const int32_t *h_ids, int n, void *cu_stream);
int mww_endpointer_reset_device(mww_endpointer_t *ep, const int32_t *d_ids, int n, void *cu_stream);
int mww_endpointer_drain(mww_endpointer_t *ep, mww_endpoint_event *h_events, int max_events, long long *n_events, void *cu_stream);
int mww_endpointer_buffers(mww_endpointer_t *ep, const long long **d_count, const mww_endpoint_event **d_events, const int32_t **d_ended,
                           const int32_t **d_armed, int *capacity);
int mww_endpointer_get_state(mww_endpointer_t *ep, mww_endpoint_state *out);
int mww_endpointer_set_state(mww_endpointer_t *ep, const mww_endpoint_state *in);
int mww_endpointer_read_commands(mww_endpointer_t *ep, mww_t *h, long long pre, long long post, int max_samples, int16_t *d_out,
                                 long long out_stride, int32_t *d_lengths, void *cu_stream);

/* ---- moving endpointer rows: export and import as packed records ----------------------------------------------------------
 * When a server moves streams to another handle (mww_export_streams, mww_export_detector_rows, mww_write_audio_history), a
 * stream that is speaking a command keeps it: its endpointer row moves as a packed device record, and the command ends with
 * the same event and the same clip as if the stream had stayed, with positions on the destination's axis.
 *   - Ids.  Both calls take GLOBAL stream ids of the endpointer's handle from host memory, as arm and reset do.  ids[i] on
 *     import may differ from the id record i was exported from, so streams can be renumbered.
 *   - One record, record_bytes long, every part padded to 16 bytes:
 *         int32   member, armed, mute, 0                member of the stream set; armed (the segmenter state follows);
 *                                                       the row's mute word from a positioned exporter, else 0
 *         int32   elapsed, run, silence, heard          zero unless armed
 *         int64   seen; uint64 flags                    VAD count and the last 64 speech flags
 *         int64   start_age, speech_end_age             S' - start_sample, S' - speech_end_sample; zero unless armed
 *         float32 hist[vad_window - 1]                  oldest first (no bytes when vad_window = 1)
 *     with S' the exporter's baseline samples_seen (its handle's counter at the endpointer's last update or whole reset).  A
 *     rule of vad_window 5 has 80-byte records: 16 + 16 + 16 + 16 + 16 (4 floats).
 *   - mww_endpointer_layout: record_bytes, vad_window, stride, hop_samples and the baseline buffered and pending rows that
 *     import checks, and the exporter's baseline samples_seen and steps, for information.  pad is 1 when the exporter is
 *     positioned (its records carry mute words) and 0 otherwise; import refuses any other value.  mww_get_endpointer_layout fills
 *     it without device work; export fills it too (out may be NULL).
 *   - export writes one record per listed id (an id may appear twice): an id that is not a member of the model's stream set
 *     gets a zero record (member = 0), an unarmed row a zero segmenter.  The endpointer does not change.
 *   - import, per listed id: a non-member of the destination's set ignores the record; a member whose record has member = 0
 *     gets what reset(ids) gives; a member whose record has member = 1 takes the record, with armed = the destination's
 *     global id when the record is armed, and positions rebased to S'_dst - age.  arm_tag is not carried (each row keeps its
 *     own).  Rows that are not listed keep every byte.  Events and d_ended do not move: drain the source first.
 *   - Time axis.  Export and import are refused unless the endpointer is up to date with its handle: the handle's
 *     samples_seen, frontend_buffered and model k's pending rows equal the endpointer's baseline (update the endpointer after
 *     the handle's last call).  Import is refused when the records' vad_window, stride, hop_samples, buffered, pending or
 *     record_bytes differ from the destination's; the message names the field.  Equal buffered and pending rows make a
 *     step's age the same on both axes; two handles serving 480-sample live calls always meet it.  Other rule fields may
 *     differ, and the row continues under the destination's rule.
 *   - Positions after the move may be negative, when the destination's axis is younger than the moved command.  The command
 *     read already handles that: it writes zeros only outside [samples_seen - C, samples_seen), and a history written with
 *     mww_write_audio_history puts the moved samples at the matching positions.
 *   - Replay limit.  A moved row's flags carry verbatim, but an arm after the move replays at most min(lookback_steps, steps
 *     the DESTINATION endpointer consumed since create or its last whole reset), as for every row there.  For a full-depth
 *     replay of a stream moved between its detection and its arm, update the destination endpointer for at least
 *     lookback_steps calls before the move (it can run on the destination handle's idle streams).
 *   - Both calls are asynchronous and ordered on cu_stream, with records [n][record_bytes] in memory the endpointer's GPU
 *     can address, 16-byte aligned.  One launch each whatever n is; n == 0 launches nothing and still fills / checks the
 *     layout.  The id list is staged in a buffer the endpointer owns, so calls on one endpointer from different CUDA streams
 *     must be ordered by the caller.
 *   - MWW_EINVAL before any device work, with the endpointer unchanged: a NULL endpointer, the conditions above, n < 0, NULL
 *     or misaligned records with n > 0, a NULL layout on import, an id out of range, an id listed twice on import. */
typedef struct mww_endpointer_layout {
    int64_t record_bytes;
    int32_t vad_window, stride, hop_samples, buffered, pending, pad;
    int64_t samples_seen, steps;      /* the exporter's baseline, for information */
} mww_endpointer_layout;
int mww_get_endpointer_layout(const mww_endpointer_t *ep, mww_endpointer_layout *out);
int mww_export_endpointer_rows(mww_endpointer_t *ep, const int32_t *h_ids, int n, void *d_records, mww_endpointer_layout *out,
                               void *cu_stream);
int mww_import_endpointer_rows(mww_endpointer_t *ep, const int32_t *h_ids, int n, const void *d_records,
                               const mww_endpointer_layout *layout, void *cu_stream);

/* ---- positioned arm: the command starts at the detection, after the wake word ----------------------------------------------
 * arm replays the row's last lookback_steps flags, which reach back over the wake word: the VAD hears it as speech, so the
 * command's clip holds the wake word, and a pause after it longer than silence_steps ends the command before it is spoken.
 * A timed detector knows where the wake word ended (its event positions, "event positions"), on the axis the endpointer's
 * steps use.  arm_at starts the command there.
 *
 * Rule.  arm_at(ids, positions, skip), for each listed id whose row r is a member; P is the id's position and skip >= 0 is in
 * samples.
 *   - Newest position.  q = S' - b' - hop g', from the endpointer's baseline (S' samples_seen, b' = buffered' - (480 - hop),
 *     g' the model's pending rows): the position of the newest step consumed, or, with no step since a whole reset, where it
 *     would have been.  Future steps fall at q + k stride hop, k >= 1.  P' = min(P, q): a position in the future counts as now.
 *   - Fresh segment.  The row gets fresh segmenter state with start_sample = speech_end_sample = P'.  The plain rule's "the
 *     first step sets start_sample" does not apply to it.
 *   - Replay.  Of arm's replay steps (L = min(lookback_steps, steps consumed)), those at p > P' run, oldest first, each with
 *     flag f' = f && p > P' + skip.  The stored flags do not change.  elapsed counts the steps replayed only: steps after P'
 *     older than the replay are not counted.  A replay that reaches an end emits its event during the call, as arm's does.
 *   - Mute.  The row keeps mute = max(0, floor((P' + skip - q) / (stride hop))): the future steps that still fall within the
 *     skip.  While the row is armed, each update step with mute > 0 takes f' = 0, then mute -= 1.
 *   - Clearing.  Every call that gives a row fresh segmenter state sets its mute to 0: arm, disarm, reset, an end, and an
 *     import of a record without a mute.
 *   - Repeated ids.  An id listed twice in one call arms once, at the latest P (equal positions give equal results): a
 *     detector may hold two slots for one stream, two fires between polls or two wake words of a models detector.
 *   - Ids.  Host ids outside [0, n_streams) are MWW_EINVAL.  Device ids that are -1, out of range or not members are ignored,
 *     as arm_device ignores them, so a verifier's d_confirmed, a guard's d_passed or a detector's d_fired go in slot for slot
 *     with the detector's d_positions (mww_get_detector_positions).
 *   - Properties.  (1) With P = (the oldest replayed position - stride hop) and skip = 0, arm_at is arm, bit for bit.  (2)
 *     Results do not depend on when arm_at is called, as long as P <= q and the replay still reaches P (its oldest step is at
 *     most P + stride hop).  (3) With every mute at 0, the positioned forms below give exactly what the plain ones give.
 *   - Command read, unchanged: a = start_sample - pre.  With pre = 0 the clip starts at the detection and leaves the wake word
 *     out; pre > 0 takes it back in.
 *
 * The mute word.  mww_endpointer_get_mutes / _set_mutes read and write every row's int32 mute word, [n_rows], synchronously,
 * beside get_state / set_state for checkpoints.  Bits 0 .. 29 hold the mute count (at most 2^22); bit 30 (placed) is set
 * while a row that arm_at armed with no step replayed has taken no step since: its start_sample is fixed, and its first step
 * leaves it.  The first step clears the bit.  set refuses a negative word or a count above 2^22.
 *
 * Mode.  An endpointer runs the plain kernels (libmww_endpoint.so, libmww_serving_records.so) and issues exactly the launches
 * it issued before this section existed, until its first arm_at, set_mutes or import of records whose layout has pad = 1.
 * From then on, for good, update, arm, disarm, reset, export and import run the positioned forms (libmww_endpoint_at.so),
 * one launch each as before; arm_at is two launches whatever n is, a reduction of each row's latest position and the arm.
 * A positioned exporter writes each armed row's mute word into its record head's third word and sets the layout's pad to 1;
 * a plain endpointer's records are byte for byte what they were.  Importing records of either kind into a positioned
 * endpointer takes the word (0 from plain records); importing positioned records into a plain endpointer makes it positioned,
 * so a mute is never dropped.
 *
 * Calls.  Asynchronous on cu_stream, no allocation: the mute words, the reduction's keys and the staging of a host list are
 * allocated at create.  A host list is copied into buffers the endpointer owns, so calls on one endpointer from different
 * CUDA streams must be ordered by the caller.  Refusals, MWW_EINVAL before any device work: a NULL endpointer, n < 0, NULL
 * ids or positions with n > 0, skip_samples outside [0, 2^22], and a host id out of range. */
int mww_endpointer_arm_at(mww_endpointer_t *ep, const int32_t *h_ids, const int64_t *h_positions, int n, long long skip_samples, void *cu_stream);
int mww_endpointer_arm_at_device(mww_endpointer_t *ep, const int32_t *d_ids, const int64_t *d_positions, int n, long long skip_samples,
                                 void *cu_stream);
int mww_endpointer_get_mutes(mww_endpointer_t *ep, int32_t *h_mutes);
int mww_endpointer_set_mutes(mww_endpointer_t *ep, const int32_t *h_mutes);

#ifdef __cplusplus
}
#endif
#endif /* MWW_H_ */
