// mww_capi.cu -- the extern "C" boundary declared in include/mww.h.
//
// Host-side orchestration only: weight/table upload (container parsing: mww_container.cc), per-stream state,
// stream tiling against a scratch budget, and the pipelined host-buffer path.  All arithmetic is
// in the kernels (mww_frontend.cu, mww_nn.cu, mww_nn_int8.cu); there is no CPU fallback.  The streaming detectors'
// entry points, which reach a handle only through the calls declared in include/mww.h, are in mww_detector_capi.cu.
#include <cuda_runtime.h>
#include <sched.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/syscall.h>
#include <unistd.h>

#include <algorithm>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/mww.h"
#include "mww_capi.h"
#include "mww_container.h"
#include "mww_frontend_dev.cuh"
#include "mww_history.h"
#include "mww_kernels.h"
#include "mww_nn_tc.h"
#include "mww_streams.h"

using namespace mww;

namespace {

thread_local std::string g_create_error;

constexpr int kMaxModels = 64;      // models one handle can carry (mww_create_multi)

// the streams one model runs on (mww_create_multi_streams / mww_set_model_streams): strictly increasing global ids; the
// model's state, pending rows and probabilities are indexed by position in this list (the compact index)
struct Members {
    std::vector<int32_t> ids;
    int32_t *d_ids = nullptr;       // device copy of ids (the row gather reads it)
    int32_t *d_inv = nullptr;       // [n_streams]: compact index of each global stream id, -1 for a non-member (reset by id)
};

// one NN model the frontend feeds: its weights (mww_container.h), per-stream ring state and pending rows
struct Model : ModelWeights {
    uint64_t model_hash = 0;        // FNV-1a of the model container: mww_copy_nn_state only moves state between equal models
    void *d_weights = nullptr;      // the arena of ModelWeights
    Members mem;
    void *d_nn_state = nullptr;     // float or int8 [M][G.state_elems]   (4176 for okay_nabu; M = members)
    void *d_pend = nullptr;         // float or int8 [M][G.pend_cap][40]  (2 rows for stride 3)
    int n_pend = 0;
    // live-step path: rings stay rotated between live calls (mww_nn_live.cuh); all streams advance in lockstep
    LiveHeads live_heads{};
    // every carried first-conv ring / pending row is a feature (<= 2048) x 0.0390625: true after a full reset and after a predict
    // call of >= kTcFreshSteps steps; false after infer_features (rows of any value); checked on a state set from outside
    // (note_state_set).  The fp16 first conv needs it.
    bool tc_rows_bounded = true;

    size_t elem_size() const { return quantized() ? 1 : 4; }
    int members() const { return (int)mem.ids.size(); }
    size_t state_bytes() const { return (size_t)G.state_elems * elem_size(); }                   // per stream
    size_t pend_bytes() const { return (size_t)G.pend_cap * kNumChannels * elem_size(); }       // per stream
    // compact index `first`'s ring state and pending rows
    template <typename T> T *state(int first) const { return static_cast<T *>(d_nn_state) + (size_t)first * G.state_elems; }
    template <typename T> T *pend(int first) const { return static_cast<T *>(d_pend) + (size_t)first * G.pend_cap * kNumChannels; }
};

// the streams of one input rate of a handle with per-stream rates (mww_set_stream_rates): the rate's plan and polyphase
// table, and its members, rate_ids[off, off + n) (sorted)
constexpr int kNumRates = (int)(sizeof kResampleRates / sizeof kResampleRates[0]);
struct RateGroup {
    ResamplePlan P;
    int16_t *d_table = nullptr;     // [L][pitch]; none at 16 kHz (the identity plan)
    int off = 0, n = 0;
};

}  // namespace

struct mww_handle {
    int device = 0, n_streams = 0, sm_count = 132;
    std::string err;
    // constant tables
    uint8_t *d_tables = nullptr;
    FrontendParams P;
    bool no_tc = false;             // MWW_NO_TC: keep the mma.sync clip kernel (A/B measurements)
    int live_variant = 3;           // MWW_LIVE_VARIANT: 3 = bulk-copy stages (default), 2 = warp-specialised with register loads, 1 = r01 kernel
    // per-stream frontend state
    int16_t *d_carry = nullptr;
    uint32_t *d_estimate = nullptr;
    int used = 0;
    int hop = kHop;                 // samples between feature windows (mww_set_window_step; 160 = the 10 ms of every shipped model)
    // input-rate resampler (mww_set_input_rate; mww_resample.h): none at 16 kHz
    ResamplePlan rs;
    int16_t *d_rs_table = nullptr;  // [L][pitch]
    int16_t *d_rs_hist = nullptr;   // [n_streams][rs_hist_stride], the first H samples of each row used
    int rs_hist_stride = 0;         // H rounded up to even: whole 4-byte words per stream (reset by id)
    long long rs_seen = 0;          // input samples every stream has been given since the last full / frontend reset
    int16_t *d_rs_out = nullptr; size_t rs_out_bytes = 0;     // one tile's 16 kHz samples
    // per-stream rates (mww_set_stream_rates): rs stays the 16 kHz plan, rs_seen counts t (16 kHz samples every stream has
    // been given), d_rs_hist rows hold resample_max_history() samples, and each rate has its table and member list
    bool per_rate = false;
    std::vector<int32_t> stream_rate;                   // [n_streams]
    RateGroup groups[kNumRates];
    std::vector<int32_t> rate_ids;                      // every group's members, group after group
    int32_t *d_rate_ids = nullptr;                      // device copy of rate_ids
    // per-stream sample formats (mww_set_stream_formats) of the _mixed entry points: each stream's kFormat* code, its device
    // copy, and per rate the formats (bit f for code f) of that rate's members
    std::vector<uint8_t> stream_format;                 // [n_streams]
    uint8_t *d_stream_format = nullptr;
    unsigned rate_formats[kNumRates] = {};
    // audio history (mww_set_audio_history; mww_history.h): the last hist_cap 16 kHz samples of every stream, a ring row per
    // stream; hist_seen counts the samples appended since it was enabled (resets zero rows, not the counter)
    int16_t *d_hist = nullptr;                          // [n_streams][hist_cap]
    int hist_cap = 0;
    long long hist_seen = 0;
    // scratch
    uint32_t *d_v = nullptr; size_t v_bytes = 0;
    uint16_t *d_feat = nullptr; size_t feat_bytes = 0;
    uint16_t *d_gather = nullptr; size_t gather_bytes = 0;     // one tile's rows of one model whose members are not consecutive
    int32_t *d_cids = nullptr; size_t cids_cap = 0;            // reset by id: the ids translated to one model's compact indices
    size_t scratch_budget = (size_t)2048 << 20;
    int min_tile_streams = 2048;       // staged path: a tile never gets fewer streams than this (MWW_MIN_TILE_STREAMS)
    // host-buffer pipeline
    cudaStream_t st_h2d = nullptr, st_compute = nullptr, st_d2h = nullptr;
    cudaEvent_t ev_h2d[2] = {nullptr, nullptr}, ev_compute[2] = {nullptr, nullptr}, ev_d2h[2] = {nullptr, nullptr};
    cudaEvent_t ev_entry = nullptr, ev_exit = nullptr;
    bool staged_used = false;      // ev_compute[] have been recorded by an earlier staged call
    bool poisoned = false;         // a staged call failed half-way: per-stream state is inconsistent until mww_reset(all)
    int32_t *d_ids = nullptr; size_t ids_cap = 0;      // device copy of a host id list (mww_reset)
    void *d_audio_tile[2] = {nullptr, nullptr}; size_t audio_tile_bytes = 0;     // int16 or float32 samples of one tile
    float *d_probs_tile[2] = {nullptr, nullptr}; size_t probs_tile_bytes = 0;
    bool no_live = false, no_fuse = false;
    long long launches = 0;
    // the NN models the frontend feeds: one for mww_create with a model, none for a frontend-only handle, K for mww_create_multi
    std::vector<Model> models;
    // optional per-kernel timing (mww_profile_*)
    bool profiling = false;
    std::vector<cudaEvent_t> prof_ev[4];   // start/stop pairs per kernel class
    std::vector<cudaEvent_t> tl_ev;        // last staged call while profiling: 4 events per tile (mww_timeline_read)
};

int mww::fail(mww_t *h, int code, const std::string &msg) {
    if (h) h->err = msg; else g_create_error = msg;
    return code;
}
int mww::cuda_fail(mww_t *h, cudaError_t e, const char *what) {
    return fail(h, MWW_ECUDA, std::string(what) + ": " + cudaGetErrorString(e));
}

namespace {

#define CU(h, call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return cuda_fail(h, e_, #call); } while (0)
#define ENTER(h) DeviceGuard guard_((h)->device); if (guard_.err != cudaSuccess) return cuda_fail((h), guard_.err, "cudaSetDevice")
#define ENTER_STATEFUL(h) ENTER(h); if ((h)->poisoned) return fail((h), MWW_ECUDA, "an earlier staged call failed half-way; per-stream state is inconsistent until mww_reset(h, NULL, 0, stream)")

// RAII bracket: records an event pair around a launch when profiling is on
struct ProfScope {
    mww_t *h; int cls; cudaStream_t st; cudaEvent_t stop = nullptr;
    ProfScope(mww_t *h_, int cls_, cudaStream_t st_) : h(h_), cls(cls_), st(st_) {
        if (!h->profiling) return;
        cudaEvent_t a = nullptr;
        if (cudaEventCreate(&a) != cudaSuccess || cudaEventCreate(&stop) != cudaSuccess) { stop = nullptr; return; }
        cudaEventRecord(a, st);
        h->prof_ev[cls].push_back(a);
        h->prof_ev[cls].push_back(stop);
    }
    ~ProfScope() { if (stop) cudaEventRecord(stop, st); }
};

int ensure_scratch(mww_t *h, size_t v_bytes, size_t feat_bytes, size_t gather_bytes = 0) {
    if (gather_bytes > h->gather_bytes) {
        if (h->d_gather) cudaFree(h->d_gather);
        h->d_gather = nullptr; h->gather_bytes = 0;
        CU(h, cudaMalloc(&h->d_gather, gather_bytes));
        h->gather_bytes = gather_bytes;
    }
    if (v_bytes > h->v_bytes) {
        if (h->d_v) cudaFree(h->d_v);
        h->d_v = nullptr; h->v_bytes = 0;
        CU(h, cudaMalloc(&h->d_v, v_bytes));
        h->v_bytes = v_bytes;
    }
    if (feat_bytes > h->feat_bytes) {
        if (h->d_feat) cudaFree(h->d_feat);
        h->d_feat = nullptr; h->feat_bytes = 0;
        CU(h, cudaMalloc(&h->d_feat, feat_bytes));
        h->feat_bytes = feat_bytes;
    }
    return MWW_OK;
}

bool resampling(const mww_t *h) { return h->per_rate || h->rs.rate != 16000; }
// 16 kHz samples a call of n input-rate samples gives every stream (per-stream rates: n is n16 already)
int samples16(const mww_t *h, int n) {
    return h->per_rate ? n : (resampling(h) ? resample_call_outputs(h->rs_seen, n, h->rs.L, h->rs.M) : n);
}
// per-stream rates: the input samples a call of n16 takes from each stream of group g, N(t + n16) - N(t)
long long rate_inputs(const mww_t *h, const RateGroup &g, int n16) {
    return resample_inputs(h->rs_seen + n16, g.P.L, g.P.M) - resample_inputs(h->rs_seen, g.P.L, g.P.M);
}
// the samples a row of the caller's audio holds for a call of n: n, or per-stream rates the largest D_s of any rate present
long long input_width(const mww_t *h, int n) {
    if (!h->per_rate || n <= 0) return n;
    long long w = 0;
    for (const RateGroup &g : h->groups)
        if (g.n > 0) w = std::max(w, rate_inputs(h, g, n));
    return w;
}
// the resampler's index math is int32 in upsampled samples: a call must keep n L below 2^31 (about 100 s at 22.05 kHz), at
// every rate present
bool resample_call_fits(const mww_t *h, int n) {
    if (h->per_rate) {
        for (const RateGroup &g : h->groups)
            if (g.n > 0 && rate_inputs(h, g, n) * g.P.L + g.P.M >= (1ll << 31)) return false;
        return true;
    }
    return !resampling(h) || (long long)n * h->rs.L + h->rs.M < (1ll << 31);
}
// the audio arguments every audio entry point checks first.  Per-stream rates: n_samples is n16 and must be even, and each
// row must hold the call's largest D_s.
bool bad_audio(const mww_t *h, int n_samples, const void *audio, long long audio_stride) {
    return n_samples < 0 || (h->per_rate && (n_samples & 1)) || (n_samples > 0 && !audio) || audio_stride < input_width(h, n_samples);
}
// Mixed byte rows (the _mixed entry points, per-stream rates only): row s holds D_s samples of stream s's format.  The call's
// widest row over the (rate, format) pairs present, in bytes.
long long mixed_width(const mww_t *h, int n16) {
    long long w = 0;
    for (int i = 0; i < kNumRates; ++i)
        for (int f = 0; f < kNumFormats; ++f)
            if (h->groups[i].n > 0 && (h->rate_formats[i] >> f & 1)) w = std::max(w, rate_inputs(h, h->groups[i], n16) * format_bytes(f));
    return w;
}
// the same over streams [first, first + n) only: the bytes the staged paths copy per row of that tile
long long mixed_tile_width(const mww_t *h, int first, int n, int n16) {
    if (first == 0 && n == h->n_streams) return mixed_width(h, n16);
    return mixed_rows_width(h->stream_rate.data(), h->stream_format.data(), first, n, h->rs_seen, n16);
}
// the audio arguments of a mixed call: n16 as bad_audio, and the base and the byte stride multiples of 4 (float rows
// aligned), the stride at least the widest row.  The caller has checked that the handle has per-stream rates.
bool bad_audio(const mww_t *h, int n_samples, const Mixed8 *audio, long long audio_stride) {
    return n_samples < 0 || (n_samples & 1) || (n_samples > 0 && !audio) || audio_stride < mixed_width(h, n_samples) || (audio_stride & 3) ||
           (reinterpret_cast<uintptr_t>(audio) & 3);
}
// Mixed rows reach only the resampler: the _mixed entry points refuse a handle without per-stream rates before anything
// else, and on a handle with them every kernel after the resampler reads the 16 kHz scratch.  The call bodies name the
// direct paths of a single-rate handle for every sample type; with mixed rows they are never taken.
int mixed_direct(mww_t *h) { return fail(h, MWW_EUNSUPPORTED, "mixed rows need per-stream rates"); }
// the samples (for mixed rows the bytes) a row of the caller's audio holds for a call of n
template <typename T>
long long row_width(const mww_t *h, int n) {
    if constexpr (std::is_same<T, Mixed8>::value) return mixed_width(h, n);
    else return input_width(h, n);
}

// samples of the resampler history a stream keeps (the row length of mww_get_resampler_state)
int hist_len(const mww_t *h) { return h->per_rate ? resample_max_history() : h->rs.H; }

int ensure_rs_out(mww_t *h, size_t bytes) {
    if (bytes <= h->rs_out_bytes) return MWW_OK;
    if (h->d_rs_out) cudaFree(h->d_rs_out);
    h->d_rs_out = nullptr; h->rs_out_bytes = 0;
    CU(h, cudaMalloc(&h->d_rs_out, bytes));
    h->rs_out_bytes = bytes;
    return MWW_OK;
}

// streams [first, first + n) of a call of n_in input-rate samples -> their n16 16 kHz samples in h->d_rs_out [n][n16], each
// stream's history moved on.  One launch; the caller advances h->rs_seen once the whole call is issued.
// Per-stream rates: one launch per rate with members in the tile [first, first + n), over those members only; the 16 kHz
// members' samples are copied (the identity plan).
template <typename T>
int run_rates_tile(mww_t *h, int first, int n, const T *d_audio, long long audio_stride, int n16, cudaStream_t st) {
    for (const RateGroup &g : h->groups) {
        int a = 0, b = 0;
        tile_members(h->rate_ids.data() + g.off, g.n, first, n, &a, &b);
        const int n_in = (int)rate_inputs(h, g, n16);      // below 2^31 / L: resample_call_fits
        if (b == a || n_in <= 0) continue;
        ResampleArgs r;
        r.table = g.d_table; r.hist = h->d_rs_hist; r.hist_stride = h->rs_hist_stride;
        r.audio_stride = audio_stride; r.out_stride = n16;
        r.L = g.P.L; r.M = g.P.M; r.T = g.P.T; r.H = g.P.H; r.pitch = g.P.pitch;
        r.t0 = resample_t0(resample_inputs(h->rs_seen, g.P.L, g.P.M), g.P.L, g.P.M); r.n_in = n_in; r.n_out = n16; r.n_streams = b - a;
        if constexpr (std::is_same<T, Mixed8>::value)
            CU(h, launch_resample_mixed(r, h->d_rate_ids + g.off + a, first, h->d_stream_format, d_audio, h->d_rs_out, h->sm_count, st));
        else
            CU(h, launch_resample_members(r, h->d_rate_ids + g.off + a, first, d_audio, h->d_rs_out, h->sm_count, st));
        h->launches += 1;
    }
    return MWW_OK;
}

template <typename T>
int run_resample_tile(mww_t *h, int first, int n, const T *d_audio, long long audio_stride, int n_in, int n16, cudaStream_t st) {
    if (h->per_rate) return run_rates_tile(h, first, n, d_audio, audio_stride, n16, st);
    if constexpr (std::is_same<T, Mixed8>::value) {
        return mixed_direct(h);
    } else {
        if (n_in <= 0) return MWW_OK;
        ResampleArgs a;
        a.table = h->d_rs_table; a.hist = h->d_rs_hist + (size_t)first * h->rs_hist_stride; a.hist_stride = h->rs_hist_stride;
        a.audio_stride = audio_stride; a.out_stride = n16;
        a.L = h->rs.L; a.M = h->rs.M; a.T = h->rs.T; a.H = h->rs.H; a.pitch = h->rs.pitch;
        a.t0 = resample_t0(h->rs_seen, h->rs.L, h->rs.M); a.n_in = n_in; a.n_out = n16; a.n_streams = n;
        CU(h, launch_resample(a, d_audio, h->d_rs_out, h->sm_count, st));
        h->launches += 1;
        return MWW_OK;
    }
}

int frames_for(const mww_t *h, int n_samples) {
    const long long total = (long long)h->used + n_samples;
    return total >= kWindow ? (int)((total - kWindow) / h->hop + 1) : 0;
}

// Long calls over enough streams run K1 + the temporal chain in one kernel (one CTA per stream) and need no K1->K2 scratch.
bool clip_fuses(const mww_t *h, int n_frames) {
    return h->hop != kHop || (!h->no_fuse && frontend_clip_fuses(h->n_streams, n_frames, h->sm_count));     // the run-time-hop kernel is always fused
}
size_t v_scratch_bytes(const mww_t *h, int tile, int n_frames) {
    return clip_fuses(h, n_frames) ? 0 : (size_t)tile * std::max(n_frames, 1) * kNumChannels * 4;
}

// streams per tile so that the K1->K2 scratch (when the call needs one), the optional feature scratch and `extra_per_stream`
// further bytes of each stream fit the budget
int tile_streams(const mww_t *h, int n_frames, bool need_feat, size_t extra_per_stream = 0) {
    const size_t per_stream = (size_t)std::max(n_frames, 1) * kNumChannels * ((clip_fuses(h, n_frames) ? 0 : 4) + (need_feat ? 2 : 0)) +
                              extra_per_stream;
    if (per_stream == 0) return h->n_streams;
    size_t t = h->scratch_budget / per_stream;
    if (t < 1) t = 1;
    if (t > (size_t)h->n_streams) t = (size_t)h->n_streams;
    return (int)t;
}

// Bytes per stream of the row-gather buffer a predict call needs: none while every model's members are consecutive stream
// ids (all streams, or one block), so such handles keep the tiles and launches of a handle without stream sets.
size_t gather_bytes_per_stream(const mww_t *h, int n_frames) {
    for (const Model &m : h->models) {
        const std::vector<int32_t> &ids = m.mem.ids;
        if (!ids.empty() && ids.back() - ids.front() != (int)ids.size() - 1) return (size_t)std::max(n_frames, 1) * kNumChannels * 2;
    }
    return 0;
}

// frontend for streams [first, first+n): audio tile pointer is already offset to the tile's first stream.  T = int16_t or
// float (converted to int16 inside the kernels); everything after the frontend is the same for both.
template <typename T>
int run_frontend_tile(mww_t *h, int first, int n, const T *d_audio, long long audio_stride, int n_samples,
                      int n_frames, uint16_t *d_feat, long long feat_stream_stride, cudaStream_t st) {
    if (n_frames <= 0) return MWW_OK;
    if (h->hop != kHop) {
        ProfScope p(h, 0, st);
        CU(h, launch_frontend_hop(h->P, h->d_carry + (size_t)first * kWindow, h->used, d_audio, audio_stride, n_samples, n, n_frames, h->hop,
                                  h->d_estimate + (size_t)first * kNumChannels, d_feat, feat_stream_stride, st));
        h->launches += 1;
        return MWW_OK;
    }
    if (!h->no_fuse && frontend_fusable(h->used, n_samples, n_frames)) {
        // short call: K1 + K2 + carry update in one launch (run_carry_tile sees the same predicate and does nothing)
        ProfScope p(h, 0, st);
        CU(h, launch_frontend_fused(h->P, h->d_carry + (size_t)first * kWindow, h->used, d_audio, audio_stride, n_samples, n,
                                    n_frames, h->d_estimate + (size_t)first * kNumChannels, d_feat, feat_stream_stride, st));
        h->launches += 1;
        return MWW_OK;
    }
    if (clip_fuses(h, n_frames)) {
        // long call, one CTA per stream: K1 and the temporal chain in one launch, features written directly (whatever the
        // size of this particular tile -- the scratch was sized for the fused form).  k1_clip_kernel, with half-warp barriers;
        // MWW_K1_OCC=3 (read once per process) selects the 3-CTA-per-SM kernel with its lane twiddles in registers.
        static const bool occ3 = getenv("MWW_K1_OCC") != nullptr && atoi(getenv("MWW_K1_OCC")) == 3;
        ProfScope p(h, 0, st);
        if (occ3)
            CU(h, launch_frontend_clip_fused(h->P, h->d_carry + (size_t)first * kWindow, h->used, d_audio, audio_stride, n_samples, n, n_frames,
                                             h->d_estimate + (size_t)first * kNumChannels, d_feat, feat_stream_stride, st));
        else
            CU(h, launch_frontend_clip(h->P, h->d_carry + (size_t)first * kWindow, h->used, d_audio, audio_stride, n_samples, n, n_frames,
                                       h->d_estimate + (size_t)first * kNumChannels, d_feat, feat_stream_stride, st));
        h->launches += 1;
        return MWW_OK;
    }
    {
        ProfScope p(h, 0, st);
        CU(h, launch_k1(h->P, h->d_carry + (size_t)first * kWindow, h->used, d_audio, audio_stride, n_samples, n,
                        n_frames, h->d_v, h->sm_count, st));
    }
    {
        ProfScope p(h, 1, st);
        CU(h, launch_k2(h->P, h->d_v, n, n_frames, h->d_estimate + (size_t)first * kNumChannels, d_feat, feat_stream_stride, st));
    }
    h->launches += 2;
    return MWW_OK;
}

template <typename T>
int run_carry_tile(mww_t *h, int first, int n, const T *d_audio, long long audio_stride, int n_samples, int n_frames,
                   cudaStream_t st) {
    const int consumed = n_frames * h->hop;
    const int new_used = h->used + n_samples - consumed;
    if (h->hop == kHop && !h->no_fuse && n_frames > 0 && frontend_fusable(h->used, n_samples, n_frames)) return MWW_OK;     // done by the fused frontend kernel
    ProfScope p(h, 3, st);
    CU(h, launch_carry_update(h->d_carry + (size_t)first * kWindow, h->used, d_audio, audio_stride, n_samples, n, consumed, new_used, st));
    h->launches += 1;
    return MWW_OK;
}

// the audio history of streams [first, first + n): the call's n16 16 kHz samples from the source the carry update reads.
// Unlike the carry update it runs after the fused short-call kernel too.  The caller advances h->hist_seen once per call.
template <typename T>
int run_history_tile(mww_t *h, int first, int n, const T *d_audio, long long audio_stride, int n16, cudaStream_t st) {
    if (!h->d_hist || n16 <= 0) return MWW_OK;
    CU(h, launch_history_append(h->d_hist + (size_t)first * h->hist_cap, h->hist_cap, h->hist_seen, d_audio, audio_stride, n16, n, h->sm_count, st));
    h->launches += 1;
    return MWW_OK;
}
// the direct paths with mixed rows: never taken (mixed_direct)
int run_frontend_tile(mww_t *h, int, int, const Mixed8 *, long long, int, int, uint16_t *, long long, cudaStream_t) { return mixed_direct(h); }
int run_carry_tile(mww_t *h, int, int, const Mixed8 *, long long, int, int, cudaStream_t) { return mixed_direct(h); }
int run_history_tile(mww_t *h, int, int, const Mixed8 *, long long, int, cudaStream_t) { return mixed_direct(h); }

// once per call, where the frontend's counters move on
void end_history_call(mww_t *h, int n16) {
    if (h->d_hist) h->hist_seen += n16;
}

// one model step per stream -> the stream-parallel live-step kernels (fp32: mww_nn_live.cuh, int8: mww_nn_i8_live.cuh)
bool use_live(const mww_t *h, const Model &m, int n_rows) { return m.compiled() && n_rows == 3 && !h->no_live; }

// rotate every ring back to the canonical layout before anything that assumes it (clip kernels, mww_get_state)
int canonicalise_rings(mww_t *h, Model &m, cudaStream_t st) {
    bool any = false;
    for (int i = 0; i < 5; ++i) any = any || m.live_heads.h[i] != 0;
    if (!any) return MWW_OK;
    if (m.members() > 0) {
        if (m.quantized()) CU(h, launch_nn_i8_live_canonicalise(m.state<int8_t>(0), m.members(), m.live_heads, st));
        else CU(h, launch_nn_live_canonicalise(m.state<float>(0), m.members(), m.live_heads, st));
        h->launches += 1;
    }
    m.live_heads = LiveHeads{};
    return MWW_OK;
}
// once per API call, around the tile loop
int begin_nn_call(mww_t *h, Model &m, int n_rows, cudaStream_t st) { return use_live(h, m, n_rows) ? MWW_OK : canonicalise_rings(h, m, st); }
void end_nn_call(mww_t *h, Model &m, int n_rows) {
    if (!use_live(h, m, n_rows)) return;
    for (int i = 0; i < 5; ++i) m.live_heads.h[i] = (m.live_heads.h[i] + 1) % kLiveRingRows[i];
}

int run_nn_tile(mww_t *h, Model &m, int first, int n, const void *d_rows, int row_type, long long rows_stream_stride_rows, int n_rows,
                float *d_probs, long long probs_stride, cudaStream_t st) {
    ProfScope p(h, 2, st);
    if (row_type != MWW_ROWS_F32 && row_type != MWW_ROWS_U16 && row_type != MWW_ROWS_I8) return fail(h, MWW_EINVAL, "unknown row_type");
    if (row_type == MWW_ROWS_I8 && !m.quantized()) return fail(h, MWW_EINVAL, "int8 rows need a quantised model (inference.py:110)");
    const long long rows_stride_bytes = rows_stream_stride_rows * kNumChannels * (row_type == MWW_ROWS_F32 ? 4 : (row_type == MWW_ROWS_U16 ? 2 : 1));
    switch (m.kind) {
    // any architecture other than the compiled-in one: run-time-geometry kernels (mww_nn_generic.cuh)
    case ModelKind::kGenericI8:
        CU(h, launch_nn_generic_i8(m.G, m.GQ, m.state<int8_t>(first), m.pend<int8_t>(first), m.n_pend, d_rows, rows_stride_bytes, n_rows, row_type,
                                   d_probs, probs_stride, n, st));
        break;
    case ModelKind::kHybrid:
        CU(h, launch_nn_generic_hybrid(m.G, m.GW, m.GH, m.state<float>(first), m.pend<float>(first), m.n_pend, d_rows, rows_stride_bytes, n_rows,
                                       row_type, d_probs, probs_stride, n, st));
        break;
    case ModelKind::kGenericF32:
        CU(h, launch_nn_generic_f32(m.G, m.GW, m.state<float>(first), m.pend<float>(first), m.n_pend, d_rows, rows_stride_bytes, n_rows, row_type,
                                    d_probs, probs_stride, n, st));
        break;
    case ModelKind::kCompiledI8:
        if (reinterpret_cast<uintptr_t>(d_rows) % 16 != 0)          // the integer kernels read rows 8 / 16 bytes at a time
            return fail(h, MWW_EINVAL, "feature rows for an int8 model must be 16-byte aligned");
        if (use_live(h, m, n_rows))
            CU(h, launch_nn_i8_live(m.Wq, m.state<int8_t>(first), m.pend<int8_t>(first), m.n_pend, d_rows, rows_stride_bytes, row_type, d_probs,
                                    probs_stride, n, m.live_heads, h->sm_count, st));
        else
            CU(h, launch_nn_i8(m.Wq, m.state<int8_t>(first), m.pend<int8_t>(first), m.n_pend, d_rows, rows_stride_bytes, n_rows, row_type, d_probs,
                               probs_stride, n, st));
        break;
    case ModelKind::kCompiledF32:
        if (use_live(h, m, n_rows))
            // exactly one model step per stream: the stream-parallel live-step kernel (HBM-bound on the ring state)
            CU(h, launch_nn_f32_live(m.W, m.state<float>(first), m.pend<float>(first), m.n_pend, d_rows, rows_stride_bytes, row_type == MWW_ROWS_F32,
                                     d_probs, probs_stride, n, m.live_heads, h->sm_count, h->live_variant, st));
        else if (!h->no_tc && row_type == MWW_ROWS_U16 && (m.n_pend + n_rows) / 3 >= kTcMinSteps && reinterpret_cast<uintptr_t>(d_rows) % 16 == 0 &&
                 rows_stride_bytes % 16 == 0)
            // long calls on raw frontend rows: time is the M dimension of wgmma (mww_nn_tc.cu)
            CU(h, launch_nn_f32_tc(m.W, m.TW, m.tc_f16 && m.tc_rows_bounded, m.state<float>(first), m.pend<float>(first), m.n_pend,
                                   static_cast<const uint16_t *>(d_rows), rows_stream_stride_rows * kNumChannels, n_rows, d_probs, probs_stride, n,
                                   h->sm_count, st));
        else
            CU(h, launch_nn_f32(m.W, m.state<float>(first), m.pend<float>(first), m.n_pend, d_rows, rows_stride_bytes, n_rows,
                                row_type == MWW_ROWS_F32, d_probs, probs_stride, nullptr, n, st));
        break;
    }
    h->launches += 1;
    return MWW_OK;
}

template <typename T>
bool upload(uint8_t *base, size_t &cursor, const void *src, size_t bytes, const T **dev_out, cudaError_t *err) {
    cursor = (cursor + 255) / 256 * 256;
    *err = cudaMemcpy(base + cursor, src, bytes, cudaMemcpyHostToDevice);
    *dev_out = reinterpret_cast<const T *>(base + cursor);
    cursor += bytes;
    return *err == cudaSuccess;
}

int upload_tables(mww_t *h) {
    HostTables t;
    build_host_tables(&t);
    if (!t.ok || t.fb_coef.size() != (size_t)kFbCoefWords) return fail(h, MWW_EINVAL, "frontend table construction failed");
    for (int s = 0; s < kFbSlots; ++s)
        if (t.fb_slot_len[s] != kFbLen[s]) return fail(h, MWW_EINVAL, "filterbank schedule differs from the trip counts the kernel was compiled for");
    const size_t total = 64 * 1024;
    CU(h, cudaMalloc(&h->d_tables, total));
    size_t cur = 0;
    cudaError_t e;
    bool ok = upload(h->d_tables, cur, t.win_pairs, sizeof t.win_pairs, &h->P.win_pairs, &e) &&
              upload(h->d_tables, cur, t.tw, sizeof t.tw, &h->P.tw, &e) &&
              upload(h->d_tables, cur, t.super_tw, sizeof t.super_tw, &h->P.super_tw, &e) &&
              upload(h->d_tables, cur, t.fb_coef.data(), t.fb_coef.size() * sizeof(int32_t), &h->P.fb_coef, &e) &&
              upload(h->d_tables, cur, &t.fb_slots[0][0], sizeof t.fb_slots, &h->P.fb_slots, &e) &&
              upload(h->d_tables, cur, t.gain_lut, sizeof t.gain_lut, &h->P.gain_lut, &e) &&
              upload(h->d_tables, cur, t.log_lut, sizeof t.log_lut, &h->P.log_lut, &e);
    if (!ok) return cuda_fail(h, e, "table upload");
    memcpy(h->P.tw2, t.tw2, sizeof h->P.tw2);
    memcpy(h->P.fb_slot_len, t.fb_slot_len, sizeof h->P.fb_slot_len);
    return MWW_OK;
}

// A stream set's host list and device copies, and NN state for its members (state stays uninitialised): what a model needs
// for a given membership.  ids == nullptr: all streams.  On failure everything it allocated is freed again.
struct MemberState {
    Members mem;
    void *d_nn_state = nullptr, *d_pend = nullptr;
    void release() { cudaFree(mem.d_ids); cudaFree(mem.d_inv); cudaFree(d_nn_state); cudaFree(d_pend); *this = MemberState{}; }
};
int alloc_members(mww_t *h, const Model &m, const int32_t *ids, int n, MemberState *out) {
    MemberState r;
    if (ids) r.mem.ids.assign(ids, ids + n);
    else for (int s = 0; s < h->n_streams; ++s) r.mem.ids.push_back(s);
    const size_t M = r.mem.ids.size(), S = (size_t)h->n_streams;
    std::vector<int32_t> inv(S, -1);
    for (size_t j = 0; j < M; ++j) inv[(size_t)r.mem.ids[j]] = (int32_t)j;
    cudaError_t a = cudaMalloc(&r.mem.d_inv, S * sizeof(int32_t));
    if (a == cudaSuccess && M > 0) a = cudaMalloc(&r.mem.d_ids, M * sizeof(int32_t));
    if (a == cudaSuccess && M > 0) a = cudaMalloc(&r.d_nn_state, M * m.state_bytes());
    if (a == cudaSuccess && M > 0) a = cudaMalloc(&r.d_pend, M * m.pend_bytes());
    if (a == cudaSuccess) a = cudaMemcpy(r.mem.d_inv, inv.data(), S * sizeof(int32_t), cudaMemcpyHostToDevice);
    if (a == cudaSuccess && M > 0) a = cudaMemcpy(r.mem.d_ids, r.mem.ids.data(), M * sizeof(int32_t), cudaMemcpyHostToDevice);
    if (a != cudaSuccess) {
        r.release();
        return fail(h, a == cudaErrorMemoryAllocation ? MWW_ENOMEM : MWW_ECUDA, std::string("state allocation: ") + cudaGetErrorString(a));
    }
    *out = std::move(r);
    return MWW_OK;
}

// weights and per-stream NN state of one model container, for its members (ids == nullptr: all streams)
int load_model(mww_t *h, Model &m, const void *model_blob, size_t n_bytes, const int32_t *ids, int n_ids) {
    uint64_t x = 1469598103934665603ull;
    for (size_t i = 0; i < n_bytes; ++i) x = (x ^ static_cast<const uint8_t *>(model_blob)[i]) * 1099511628211ull;
    m.model_hash = x;
    std::string msg;
    if (int rc = parse_container(static_cast<const uint8_t *>(model_blob), n_bytes, &m, &msg)) return fail(h, rc, msg);
    CU(h, cudaMalloc(&m.d_weights, m.arena.size()));
    if (cudaError_t e = cudaMemcpy(m.d_weights, m.arena.data(), m.arena.size(), cudaMemcpyHostToDevice)) return cuda_fail(h, e, "weight upload");
    m.rebase(m.d_weights);
    MemberState ms;
    if (int rc = alloc_members(h, m, ids, n_ids, &ms)) return rc;
    m.mem = std::move(ms.mem);
    m.d_nn_state = ms.d_nn_state;
    m.d_pend = ms.d_pend;
    return MWW_OK;
}

// every model runs on all streams: what the one-model entry points, which move [n_streams]-shaped NN buffers, require
bool all_streams(const mww_t *h) {
    for (const Model &m : h->models)
        if (m.members() != h->n_streams) return false;
    return true;
}

// A state set from outside keeps the fp16 first conv only if every first-conv ring row (state floats [0, 80) of a stream) it
// brings and every pending row in use is a feature u <= 2048 times 0.0390625, as the kernels leave them: a snapshot taken from
// this library continues bit for bit on the kernel it left.
bool rows_are_features(const float *v, size_t n) {
    for (size_t i = 0; i < n; ++i) {
        const float u = nearbyintf(v[i] * 25.6f);
        if (!(u >= 0.f && u <= 2048.f && u * kFeatureScale == v[i])) return false;
    }
    return true;
}
void note_state_set(mww_t *h, Model &m, const void *h_nn, const void *h_pending, int pending_rows) {
    if (!h_nn && !h_pending) return;
    bool ok = m.tc_f16 && (h_nn || m.tc_rows_bounded) && (h_pending || m.tc_rows_bounded);
    for (int s = 0; ok && s < m.members(); ++s) {
        if (h_nn) ok = rows_are_features(static_cast<const float *>(h_nn) + (size_t)s * m.G.state_elems, 2 * kNumChannels);
        if (ok && h_pending)
            ok = rows_are_features(static_cast<const float *>(h_pending) + (size_t)s * m.G.pend_cap * kNumChannels, (size_t)pending_rows * kNumChannels);
    }
    m.tc_rows_bounded = ok;
}

// fresh rings and no pending rows for every stream of one model
int zero_nn_state(mww_t *h, Model &m, cudaStream_t st) {
    const int M = m.members();
    m.n_pend = 0;
    if (M == 0) {
        // a model without members holds no state
    } else if (m.kind == ModelKind::kGenericI8) {
        CU(h, launch_gen_fill_state_i8(m.G, m.GQ, m.state<int8_t>(0), m.pend<int8_t>(0), M, nullptr, M, st));
        h->launches += 1;
    } else if (m.kind == ModelKind::kCompiledI8) {
        CU(h, launch_fill_state_i8(m.Wq, m.state<int8_t>(0), m.pend<int8_t>(0), nullptr, M, M, st));
        h->launches += 1;
    } else {
        CU(h, cudaMemsetAsync(m.d_nn_state, 0, (size_t)M * m.state_bytes(), st));
        CU(h, cudaMemsetAsync(m.d_pend, 0, (size_t)M * m.pend_bytes(), st));
    }
    m.live_heads = LiveHeads{};
    m.tc_rows_bounded = true;
    return MWW_OK;
}

int zero_frontend(mww_t *h, cudaStream_t st) {
    const size_t S = (size_t)h->n_streams;
    CU(h, cudaMemsetAsync(h->d_carry, 0, S * kWindow * sizeof(int16_t), st));
    CU(h, cudaMemsetAsync(h->d_estimate, 0, S * kNumChannels * sizeof(uint32_t), st));
    if (h->d_rs_hist) CU(h, cudaMemsetAsync(h->d_rs_hist, 0, S * h->rs_hist_stride * sizeof(int16_t), st));
    if (h->d_hist) CU(h, cudaMemsetAsync(h->d_hist, 0, S * h->hist_cap * sizeof(int16_t), st));
    h->used = 0;
    h->rs_seen = 0;
    return MWW_OK;
}

int zero_state(mww_t *h, cudaStream_t st) {
    if (int rc = zero_frontend(h, st)) return rc;
    for (Model &m : h->models)
        if (int rc = zero_nn_state(h, m, st)) return rc;
    return MWW_OK;
}

void destroy_impl(mww_t *h) {
    if (!h) return;
    DeviceGuard guard(h->device);
    for (Model &m : h->models) {
        cudaFree(m.d_weights); cudaFree(m.d_nn_state); cudaFree(m.d_pend);
        cudaFree(m.mem.d_ids); cudaFree(m.mem.d_inv);
    }
    cudaFree(h->d_tables); cudaFree(h->d_carry); cudaFree(h->d_estimate);
    cudaFree(h->d_v); cudaFree(h->d_feat); cudaFree(h->d_ids);
    cudaFree(h->d_gather); cudaFree(h->d_cids);
    cudaFree(h->d_rs_table); cudaFree(h->d_rs_hist); cudaFree(h->d_rs_out); cudaFree(h->d_rate_ids); cudaFree(h->d_hist);
    cudaFree(h->d_stream_format);
    for (RateGroup &g : h->groups) cudaFree(g.d_table);
    for (int b = 0; b < 2; ++b) {
        cudaFree(h->d_audio_tile[b]); cudaFree(h->d_probs_tile[b]);
        if (h->ev_h2d[b]) cudaEventDestroy(h->ev_h2d[b]);
        if (h->ev_compute[b]) cudaEventDestroy(h->ev_compute[b]);
        if (h->ev_d2h[b]) cudaEventDestroy(h->ev_d2h[b]);
    }
    for (int c = 0; c < 4; ++c) for (cudaEvent_t e : h->prof_ev[c]) cudaEventDestroy(e);
    if (h->st_h2d) cudaStreamDestroy(h->st_h2d);
    if (h->st_compute) cudaStreamDestroy(h->st_compute);
    if (h->st_d2h) cudaStreamDestroy(h->st_d2h);
    if (h->ev_entry) cudaEventDestroy(h->ev_entry);
    if (h->ev_exit) cudaEventDestroy(h->ev_exit);
    delete h;
}

// mww_features / mww_features_f32
template <typename T>
int features_impl(mww_t *h, const char *who, const T *d_audio, int n_samples, long long audio_stride, uint16_t *d_feat, int max_rows,
                  int *h_rows_out, void *cu_stream) {
    if (!h) return MWW_EINVAL;
    if (bad_audio(h, n_samples, d_audio, audio_stride)) return fail(h, MWW_EINVAL, std::string(who) + ": bad audio arguments");
    if (!resample_call_fits(h, n_samples)) return fail(h, MWW_EINVAL, std::string(who) + ": call too long for the resampler; split it");
    ENTER_STATEFUL(h);
    cudaStream_t st = static_cast<cudaStream_t>(cu_stream);
    const int n16 = samples16(h, n_samples);
    const int n_frames = frames_for(h, n16);
    if (n_frames > max_rows || (n_frames > 0 && !d_feat))
        return fail(h, MWW_EINVAL, std::string(who) + ": feature buffer too small for the rows this call emits");
    const int tile = tile_streams(h, n_frames, false, resampling(h) ? (size_t)n16 * 2 : 0);
    int rc = ensure_scratch(h, v_scratch_bytes(h, tile, n_frames), 0);
    if (rc == MWW_OK && resampling(h)) rc = ensure_rs_out(h, (size_t)tile * std::max(n16, 1) * 2);
    if (rc) return rc;
    for (int first = 0; first < h->n_streams; first += tile) {
        const int n = std::min(tile, h->n_streams - first);
        uint16_t *feat = d_feat + (size_t)first * max_rows * kNumChannels;
        if (resampling(h)) {
            // the tile's 16 kHz samples, then the int16 frontend and window carry on them
            if ((rc = run_resample_tile(h, first, n, d_audio + (size_t)first * audio_stride, audio_stride, n_samples, n16, st))) return rc;
            if ((rc = run_frontend_tile(h, first, n, h->d_rs_out, n16, n16, n_frames, feat, (long long)max_rows * kNumChannels, st))) return rc;
            if (n16 > 0 && (rc = run_carry_tile(h, first, n, h->d_rs_out, n16, n16, n_frames, st))) return rc;
            if ((rc = run_history_tile(h, first, n, h->d_rs_out, n16, n16, st))) return rc;
            continue;
        }
        rc = run_frontend_tile(h, first, n, d_audio + (size_t)first * audio_stride, audio_stride, n_samples, n_frames,
                               feat, (long long)max_rows * kNumChannels, st);
        if (rc) return rc;
    }
    if (n_samples > 0 && !resampling(h)) {
        rc = run_carry_tile(h, 0, h->n_streams, d_audio, audio_stride, n_samples, n_frames, st);
        if (rc == MWW_OK) rc = run_history_tile(h, 0, h->n_streams, d_audio, audio_stride, n_samples, st);
        if (rc) return rc;
    }
    h->used = h->used + n16 - n_frames * h->hop;
    if (resampling(h)) h->rs_seen += n_samples;
    end_history_call(h, n16);
    if (h_rows_out) *h_rows_out = n_frames;
    return MWW_OK;
}

// Per-model arguments of a predict call: model k writes its probabilities to probs[k] ([members][max_probs[k]]) and runs
// steps[k] model steps (its own stride and pending rows decide how many).  Checked for every model before anything is
// launched, so a too-small buffer for one model leaves the whole handle untouched; a model without members needs none.
struct NnOuts {
    float *const *probs; const int *max_probs; int steps[kMaxModels];
};
int check_outs(mww_t *h, const char *who, int n_frames, float *const *probs, const int *max_probs, NnOuts *o) {
    if (h->models.size() > 1 && (!probs || !max_probs)) return fail(h, MWW_EINVAL, std::string(who) + ": NULL output arrays");
    o->probs = probs; o->max_probs = max_probs;
    for (size_t k = 0; k < h->models.size(); ++k) {
        const Model &m = h->models[k];
        o->steps[k] = (m.n_pend + n_frames) / m.G.stride;
        if (m.members() > 0 && (o->steps[k] > max_probs[k] || (o->steps[k] > 0 && !probs[k])))
            return fail(h, MWW_EINVAL, std::string(who) + ": probability buffer too small" +
                                           (h->models.size() > 1 ? " for model " + std::to_string(k) : std::string()));
    }
    return MWW_OK;
}
// once per call, after the last tile: every model's pending rows and live ring heads move on
void end_models_call(mww_t *h, int n_frames, const NnOuts &o, int *h_probs_out) {
    for (size_t k = 0; k < h->models.size(); ++k) {
        Model &m = h->models[k];
        end_nn_call(h, m, n_frames);
        if (o.steps[k] >= kTcFreshSteps) m.tc_rows_bounded = true;      // first-conv ring, pending rows: this call's own rows
        m.n_pend = (m.n_pend + n_frames) % m.G.stride;
        if (h_probs_out) h_probs_out[k] = o.steps[k];
    }
}
int begin_models_call(mww_t *h, int n_frames, cudaStream_t st) {
    for (Model &m : h->models)
        if (int rc = begin_nn_call(h, m, n_frames, st)) return rc;
    return MWW_OK;
}
// model k's members in the stream tile [first, first + n): compact indices [a, b), consecutive stream ids or not
struct TileSpan { int a = 0, b = 0; bool consecutive = true; };
void tile_spans(const mww_t *h, int first, int n, TileSpan *span) {
    for (size_t k = 0; k < h->models.size(); ++k) {
        const Members &mem = h->models[k].mem;
        span[k].consecutive = tile_members(mem.ids.data(), (int)mem.ids.size(), first, n, &span[k].a, &span[k].b);
    }
}

// every model on one tile of frontend rows (h->d_feat, from stream `first`); probs[k] (pitch probs_stride[k]) points at the
// row of model k's first member in the tile, compact index span[k].a.  A model whose members are consecutive reads the rows
// in place -- for all streams this is exactly the one launch per model of a handle without stream sets -- any other is
// run on a gathered copy of its members' rows.  The models share one gather buffer: they run in order on one stream.
int run_models_tile(mww_t *h, int first, int n_frames, const TileSpan *span, float *const *probs, const long long *probs_stride, cudaStream_t st) {
    const long long rows_stride = (long long)n_frames * kNumChannels;
    for (size_t k = 0; k < h->models.size(); ++k) {
        Model &m = h->models[k];
        const TileSpan &s = span[k];
        if (s.b == s.a) continue;
        const uint16_t *rows = h->d_feat + (size_t)(m.mem.ids[s.a] - first) * rows_stride;
        if (!s.consecutive && n_frames > 0) {
            CU(h, launch_gather_rows(h->d_feat, m.mem.d_ids, s.a, first, s.b - s.a, n_frames, h->d_gather, h->sm_count, st));
            h->launches += 1;
            rows = h->d_gather;
        }
        if (int rc = run_nn_tile(h, m, s.a, s.b - s.a, rows, MWW_ROWS_U16, n_frames, n_frames, probs[k], probs_stride[k], st)) return rc;
    }
    return MWW_OK;
}

// mww_predict_clip[_multi] / mww_predict_clip[_multi]_f32: the frontend runs once per stream tile, then every model on its rows
template <typename T>
int predict_clip_impl(mww_t *h, const char *who, const T *d_audio, int n_samples, long long audio_stride, float *const *d_probs,
                      const int *max_probs, int *h_probs_out, void *cu_stream) {
    if (!h) return MWW_EINVAL;
    if (bad_audio(h, n_samples, d_audio, audio_stride)) return fail(h, MWW_EINVAL, std::string(who) + ": bad audio arguments");
    if (h->models.empty()) return fail(h, MWW_EINVAL, std::string(who) + ": frontend-only handle (created without a model)");
    if (!resample_call_fits(h, n_samples)) return fail(h, MWW_EINVAL, std::string(who) + ": call too long for the resampler; split it");
    ENTER_STATEFUL(h);
    cudaStream_t st = static_cast<cudaStream_t>(cu_stream);
    const int n16 = samples16(h, n_samples);
    const int n_frames = frames_for(h, n16);
    NnOuts o;
    int rc = check_outs(h, who, n_frames, d_probs, max_probs, &o);
    if (rc) return rc;
    const size_t gather = gather_bytes_per_stream(h, n_frames);
    const int tile = tile_streams(h, n_frames, true, gather + (resampling(h) ? (size_t)n16 * 2 : 0));
    rc = ensure_scratch(h, v_scratch_bytes(h, tile, n_frames), (size_t)tile * std::max(n_frames, 1) * kNumChannels * 2, (size_t)tile * gather);
    if (rc == MWW_OK && resampling(h)) rc = ensure_rs_out(h, (size_t)tile * std::max(n16, 1) * 2);
    if (rc) return rc;
    rc = begin_models_call(h, n_frames, st);
    if (rc) return rc;
    const size_t K = h->models.size();
    float *tile_probs[kMaxModels];
    long long probs_stride[kMaxModels];
    TileSpan span[kMaxModels];
    for (size_t k = 0; k < K; ++k) probs_stride[k] = max_probs[k];
    for (int first = 0; first < h->n_streams; first += tile) {
        const int n = std::min(tile, h->n_streams - first);
        if (resampling(h)) {
            rc = run_resample_tile(h, first, n, d_audio + (size_t)first * audio_stride, audio_stride, n_samples, n16, st);
            if (rc == MWW_OK) rc = run_frontend_tile(h, first, n, h->d_rs_out, n16, n16, n_frames, h->d_feat, (long long)n_frames * kNumChannels, st);
        } else {
            rc = run_frontend_tile(h, first, n, d_audio + (size_t)first * audio_stride, audio_stride, n_samples, n_frames, h->d_feat,
                                   (long long)n_frames * kNumChannels, st);
        }
        if (rc) return rc;
        tile_spans(h, first, n, span);
        for (size_t k = 0; k < K; ++k) tile_probs[k] = d_probs[k] + (size_t)span[k].a * max_probs[k];
        rc = run_models_tile(h, first, n_frames, span, tile_probs, probs_stride, st);
        if (rc) return rc;
        // a resampling handle's carry update reads the tile's 16 kHz samples, so it runs per tile
        if (resampling(h) && n16 > 0 && (rc = run_carry_tile(h, first, n, h->d_rs_out, n16, n16, n_frames, st))) return rc;
        if (resampling(h) && (rc = run_history_tile(h, first, n, h->d_rs_out, n16, n16, st))) return rc;
    }
    end_models_call(h, n_frames, o, h_probs_out);
    if (n_samples > 0 && !resampling(h)) {
        rc = run_carry_tile(h, 0, h->n_streams, d_audio, audio_stride, n_samples, n_frames, st);
        if (rc == MWW_OK) rc = run_history_tile(h, 0, h->n_streams, d_audio, audio_stride, n_samples, st);
        if (rc) return rc;
    }
    h->used = h->used + n16 - n_frames * h->hop;
    if (resampling(h)) h->rs_seen += n_samples;
    end_history_call(h, n16);
    return MWW_OK;
}

// the one-model entry points refuse a handle that carries several models: advancing the shared frontend for one model
// would leave the others' rows behind.  They also refuse a model on a subset of the streams: their NN buffers are
// [n_streams]-shaped.
int refuse_multi(mww_t *h, const char *who, const char *instead) {
    if (h && h->models.size() > 1)
        return fail(h, MWW_EINVAL, std::string(who) + ": the handle carries " + std::to_string(h->models.size()) + " models; use " + instead);
    if (h && !all_streams(h))
        return fail(h, MWW_EINVAL, std::string(who) + ": the model runs on a subset of the streams; use " + instead);
    return MWW_OK;
}

}  // namespace

extern "C" {

namespace {

mww_t *new_handle(int device, int n_streams) {
    mww_t *h = new mww_handle();
    h->device = device;
    h->n_streams = n_streams;
    cudaDeviceGetAttribute(&h->sm_count, cudaDevAttrMultiProcessorCount, device);
    h->no_live = getenv("MWW_NO_LIVE") != nullptr;
    h->no_fuse = getenv("MWW_NO_FUSE") != nullptr;
    h->no_tc = getenv("MWW_NO_TC") != nullptr;
    h->live_variant = getenv("MWW_LIVE_VARIANT") != nullptr ? atoi(getenv("MWW_LIVE_VARIANT")) : (getenv("MWW_LIVE_V2") != nullptr ? 2 : 3);
    if (const char *mb = getenv("MWW_SCRATCH_MB")) { const long v = atol(mb); if (v > 0) h->scratch_budget = (size_t)v << 20; }
    if (const char *mt = getenv("MWW_MIN_TILE_STREAMS")) { const long v = atol(mt); if (v > 0) h->min_tile_streams = (int)v; }
    return h;
}

// mww_create (n_models 0: frontend-only, 1: one model) and mww_create_multi (`multi`: messages name the failing model's index)
// ids / n_ids (may be NULL; ids[k] == NULL: all streams): each model's stream set, already validated
int create_impl(const char *who, const void *const *blobs, const size_t *n_bytes, int n_models, int device, int n_streams, mww_t **out, bool multi,
                const int32_t *const *ids = nullptr, const int *n_ids = nullptr) {
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0)
        return fail(nullptr, MWW_ECUDA, std::string("no CUDA device available (this library has no CPU fallback): ") + cudaGetErrorString(e));
    if (device < 0 || device >= count) return fail(nullptr, MWW_EINVAL, std::string(who) + ": device index out of range");
    DeviceGuard guard(device);
    if (guard.err != cudaSuccess) return cuda_fail(nullptr, guard.err, "cudaSetDevice");
    mww_t *h = new_handle(device, n_streams);
    int rc = upload_tables(h);
    for (int k = 0; rc == MWW_OK && k < n_models; ++k) {
        h->models.emplace_back();
        const bool subset = ids && ids[k];
        rc = load_model(h, h->models.back(), blobs[k], n_bytes[k], subset ? ids[k] : nullptr, subset ? n_ids[k] : 0);
        if (rc != MWW_OK && multi) h->err = "model " + std::to_string(k) + ": " + h->err;
    }
    if (rc == MWW_OK) {
        const size_t S = (size_t)n_streams;
        cudaError_t a = cudaMalloc(&h->d_carry, S * kWindow * sizeof(int16_t));
        if (a == cudaSuccess) a = cudaMalloc(&h->d_estimate, S * kNumChannels * sizeof(uint32_t));
        if (a != cudaSuccess) rc = fail(h, a == cudaErrorMemoryAllocation ? MWW_ENOMEM : MWW_ECUDA, std::string("state allocation: ") + cudaGetErrorString(a));
    }
    if (rc == MWW_OK) rc = zero_state(h, nullptr);
    if (rc == MWW_OK) { cudaError_t s = cudaDeviceSynchronize(); if (s != cudaSuccess) rc = cuda_fail(h, s, "cudaDeviceSynchronize"); }
    if (rc != MWW_OK) { g_create_error = h->err; destroy_impl(h); return rc; }
    *out = h;
    return MWW_OK;
}

}  // namespace

int mww_create(const void *model_blob, size_t n_bytes, int device, int n_streams, mww_t **out) {
    if (out) *out = nullptr;
    if (!out || n_streams < 1) return fail(nullptr, MWW_EINVAL, "mww_create: bad arguments");
    return create_impl("mww_create", &model_blob, &n_bytes, model_blob != nullptr ? 1 : 0, device, n_streams, out, false);
}

int mww_create_multi(const void *const *blobs, const size_t *n_bytes, int n_models, int device, int n_streams, mww_t **out) {
    if (out) *out = nullptr;
    if (!out || n_streams < 1 || !blobs || !n_bytes) return fail(nullptr, MWW_EINVAL, "mww_create_multi: bad arguments");
    if (n_models < 1 || n_models > kMaxModels)
        return fail(nullptr, MWW_EINVAL, "mww_create_multi: n_models must be in [1, " + std::to_string(kMaxModels) + "]");
    for (int k = 0; k < n_models; ++k)
        if (!blobs[k]) return fail(nullptr, MWW_EINVAL, "mww_create_multi: model " + std::to_string(k) + " is NULL");
    return create_impl("mww_create_multi", blobs, n_bytes, n_models, device, n_streams, out, true);
}

int mww_create_multi_streams(const void *const *blobs, const size_t *n_bytes, int n_models, int device, int n_streams,
                             const int32_t *const *ids, const int *n_ids, mww_t **out) {
    if (out) *out = nullptr;
    if (!out || n_streams < 1 || !blobs || !n_bytes) return fail(nullptr, MWW_EINVAL, "mww_create_multi_streams: bad arguments");
    if (n_models < 1 || n_models > kMaxModels)
        return fail(nullptr, MWW_EINVAL, "mww_create_multi_streams: n_models must be in [1, " + std::to_string(kMaxModels) + "]");
    for (int k = 0; k < n_models; ++k) {
        if (!blobs[k]) return fail(nullptr, MWW_EINVAL, "mww_create_multi_streams: model " + std::to_string(k) + " is NULL");
        if (ids && ids[k] && (!n_ids || n_ids[k] < 0 || n_ids[k] > n_streams || !valid_stream_set(ids[k], n_ids[k], n_streams)))
            return fail(nullptr, MWW_EINVAL, "mww_create_multi_streams: model " + std::to_string(k) +
                                                 ": stream ids must be strictly increasing and in [0, n_streams)");
    }
    return create_impl("mww_create_multi_streams", blobs, n_bytes, n_models, device, n_streams, out, true, ids, n_ids);
}

int mww_model_count(const mww_t *h) { return h ? (int)h->models.size() : 0; }

int mww_destroy(mww_t *h) { destroy_impl(h); return MWW_OK; }

const char *mww_last_error(const mww_t *h) { return h ? h->err.c_str() : g_create_error.c_str(); }

long long mww_launch_count(const mww_t *h) { return h ? h->launches : 0; }

int mww_copy_async(void *d_dst, const void *d_src, size_t bytes, void *cu_stream) {
    if (bytes == 0) return MWW_OK;
    if (!d_dst || !d_src) { g_create_error = "mww_copy_async: null pointer"; return MWW_EINVAL; }
    const cudaError_t e = cudaMemcpyAsync(d_dst, d_src, bytes, cudaMemcpyDefault, static_cast<cudaStream_t>(cu_stream));
    if (e != cudaSuccess) { g_create_error = std::string("mww_copy_async: ") + cudaGetErrorString(e); return MWW_ECUDA; }
    return MWW_OK;
}

namespace {
int ipc_fail(const char *what, cudaError_t e) {
    g_create_error = std::string(what) + ": " + cudaGetErrorString(e);
    return MWW_ECUDA;
}
}  // namespace

int mww_ipc_alloc(size_t bytes, int device, void **d_ptr, unsigned char *handle64) {
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
    if (!d_ptr || !handle64 || bytes == 0) { g_create_error = "mww_ipc_alloc: bad argument"; return MWW_EINVAL; }
    DeviceGuard guard(device);
    cudaError_t e = guard.err;
    if (e != cudaSuccess) return ipc_fail("mww_ipc_alloc: cudaSetDevice", e);
    void *p = nullptr;
    if ((e = cudaMalloc(&p, bytes)) != cudaSuccess) return ipc_fail("mww_ipc_alloc: cudaMalloc", e);
    cudaIpcMemHandle_t hd;
    if ((e = cudaIpcGetMemHandle(&hd, p)) != cudaSuccess) { cudaFree(p); return ipc_fail("mww_ipc_alloc: cudaIpcGetMemHandle", e); }
    memcpy(handle64, &hd, 64);
    *d_ptr = p;
    return MWW_OK;
}

int mww_ipc_open(const unsigned char *handle64, int device, void **d_ptr) {
    if (!d_ptr || !handle64) { g_create_error = "mww_ipc_open: bad argument"; return MWW_EINVAL; }
    DeviceGuard guard(device);
    cudaError_t e = guard.err;
    if (e != cudaSuccess) return ipc_fail("mww_ipc_open: cudaSetDevice", e);
    cudaIpcMemHandle_t hd;
    memcpy(&hd, handle64, 64);
    void *p = nullptr;
    if ((e = cudaIpcOpenMemHandle(&p, hd, cudaIpcMemLazyEnablePeerAccess)) != cudaSuccess) return ipc_fail("mww_ipc_open: cudaIpcOpenMemHandle", e);
    *d_ptr = p;
    return MWW_OK;
}

int mww_ipc_close(void *d_ptr, int device) {
    if (!d_ptr) return MWW_OK;
    DeviceGuard guard(device);
    cudaError_t e = guard.err;
    if (e == cudaSuccess) e = cudaIpcCloseMemHandle(d_ptr);
    return e == cudaSuccess ? MWW_OK : ipc_fail("mww_ipc_close", e);
}

int mww_ipc_free(void *d_ptr, int device) {
    if (!d_ptr) return MWW_OK;
    DeviceGuard guard(device);
    cudaError_t e = guard.err;
    if (e == cudaSuccess) e = cudaFree(d_ptr);
    return e == cudaSuccess ? MWW_OK : ipc_fail("mww_ipc_free", e);
}

int mww_profile_enable(mww_t *h, int on) {
    if (!h) return MWW_EINVAL;
    h->profiling = on != 0;
    return MWW_OK;
}

int mww_profile_read(mww_t *h, double *ms4, long long *counts4) {
    if (!h || !ms4 || !counts4) return MWW_EINVAL;
    ENTER(h);
    CU(h, cudaDeviceSynchronize());
    for (int c = 0; c < 4; ++c) {
        std::vector<cudaEvent_t> &v = h->prof_ev[c];
        for (size_t i = 0; i + 1 < v.size(); i += 2) {
            float ms = 0.f;
            if (cudaEventElapsedTime(&ms, v[i], v[i + 1]) == cudaSuccess) { ms4[c] += ms; counts4[c] += 1; }
            cudaEventDestroy(v[i]); cudaEventDestroy(v[i + 1]);
        }
        v.clear();
    }
    return MWW_OK;
}

int mww_timeline_read(mww_t *h, float *ms, int max_tiles, int *n_tiles) {
    if (!h || !ms || !n_tiles || max_tiles < 0) return MWW_EINVAL;
    ENTER(h);
    CU(h, cudaDeviceSynchronize());
    const int n = (int)(h->tl_ev.size() / 4);
    *n_tiles = n;
    for (int t = 0; t < n && t < max_tiles; ++t)
        for (int i = 0; i < 4; ++i) {
            float v = 0.f;
            if (cudaEventElapsedTime(&v, h->tl_ev[0], h->tl_ev[4 * t + i]) != cudaSuccess) v = -1.f;
            ms[4 * t + i] = v;
        }
    for (cudaEvent_t e : h->tl_ev) cudaEventDestroy(e);
    h->tl_ev.clear();
    return MWW_OK;
}

namespace {
void model_info(const Model &m, mww_info *o) {
    o->is_quantized = m.quantized();
    o->input_feature_slices = m.G.stride;
    o->input_scale = m.in_scale; o->input_zero_point = m.in_zp;
    o->output_scale = m.out_scale; o->output_zero_point = m.out_zp;
    o->state_bytes_per_stream = (int)(m.G.state_elems * m.elem_size());
    o->pending_rows = m.n_pend;
    o->macs_per_step = (int)m.G.macs_per_step;
}
}  // namespace

int mww_get_info(const mww_t *h, mww_info *o) {
    if (!h || !o) return MWW_EINVAL;
    memset(o, 0, sizeof *o);
    o->n_streams = h->n_streams; o->device = h->device; o->num_features = kNumChannels;
    o->frontend_buffered = h->used; o->sm_count = h->sm_count; o->hop_samples = h->hop;
    if (!h->models.empty()) {
        model_info(h->models[0], o);
    } else {                                 // a frontend-only handle reports okay_nabu's geometry, unquantised
        const GenArch &G = okay_nabu_arch();
        o->input_feature_slices = G.stride;
        o->state_bytes_per_stream = G.state_elems * 4;
        o->macs_per_step = (int)G.macs_per_step;
    }
    return MWW_OK;
}

int mww_get_model_info(const mww_t *h, int k, mww_info *o) {
    if (!h || !o || k < 0 || k >= (int)h->models.size()) return MWW_EINVAL;
    int rc = mww_get_info(h, o);             // the shared frontend's fields
    if (rc) return rc;
    model_info(h->models[k], o);
    o->n_streams = h->models[k].members();
    return MWW_OK;
}

namespace {

// 4-byte fill of one per-stream record for a list of stream ids (device memory); ids outside [0, n_streams) are skipped
__global__ void fill_by_id_kernel(uint32_t *__restrict__ base, long long words_per_stream, uint32_t value, const int32_t *__restrict__ ids,
                                  int n_ids, int n_streams) {
    const long long total = (long long)n_ids * words_per_stream;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long k = i / words_per_stream;
        const int id = ids[k];
        if (id < 0 || id >= n_streams) continue;
        base[(long long)id * words_per_stream + (i - k * words_per_stream)] = value;
    }
}

// records [0, bound) of `base`; ids outside that range are skipped
int fill_by_id(mww_t *h, void *base, size_t bytes_per_stream, const int32_t *d_ids, int n, int bound, cudaStream_t st) {
    const long long words = (long long)(bytes_per_stream / 4);
    const long long total = words * n;
    if (total <= 0) return MWW_OK;
    const unsigned blocks = (unsigned)std::min<long long>((total + 255) / 256, (long long)h->sm_count * 16);
    fill_by_id_kernel<<<blocks, 256, 0, st>>>(static_cast<uint32_t *>(base), words, 0u, d_ids, n, bound);
    CU(h, cudaGetLastError());
    h->launches += 1;
    return MWW_OK;
}

// fresh rings and pending rows for the listed compact indices of state / pend holding `bound` streams of model m's layout;
// indices outside [0, bound) are skipped
int reset_nn_by_id(mww_t *h, const Model &m, void *state, void *pend, const int32_t *d_ids, int n, int bound, cudaStream_t st) {
    int rc = MWW_OK;
    if (m.kind == ModelKind::kGenericI8) {
        CU(h, launch_gen_fill_state_i8(m.G, m.GQ, static_cast<int8_t *>(state), static_cast<int8_t *>(pend), n, d_ids, bound, st));
        h->launches += 1;
    } else if (m.kind == ModelKind::kCompiledI8) {
        CU(h, launch_fill_state_i8(m.Wq, static_cast<int8_t *>(state), static_cast<int8_t *>(pend), d_ids, n, bound, st));
        h->launches += 1;
    } else {
        // zero rings are rotation-invariant, so streams of a handle whose rings are rotated (live mode) can be reset in place
        rc = fill_by_id(h, state, m.state_bytes(), d_ids, n, bound, st);
        if (rc == MWW_OK) rc = fill_by_id(h, pend, m.pend_bytes(), d_ids, n, bound, st);
    }
    return rc;
}

// a device int32 buffer of at least n entries; growing it first waits for the work on st that may still read the old one
int ensure_ids(mww_t *h, int32_t **buf, size_t *cap, int n, cudaStream_t st) {
    if ((size_t)n <= *cap) return MWW_OK;
    if (*buf) { CU(h, cudaStreamSynchronize(st)); cudaFree(*buf); *buf = nullptr; *cap = 0; }
    const size_t want = std::max<size_t>((size_t)n, 1024);
    CU(h, cudaMalloc(buf, want * sizeof(int32_t)));
    *cap = want;
    return MWW_OK;
}
// a host id list -> h->d_ids, ordered on st
int upload_ids(mww_t *h, const int32_t *h_ids, int n, cudaStream_t st) {
    if (int rc = ensure_ids(h, &h->d_ids, &h->ids_cap, n, st)) return rc;
    CU(h, cudaMemcpyAsync(h->d_ids, h_ids, (size_t)n * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    return MWW_OK;
}

// fresh state for the listed global stream ids: a handful of launches whatever the length of the list.  A model on all
// streams takes the ids as they are; any other first has them translated to its compact indices (-1 for a non-member,
// which the fill kernels skip).
int reset_by_id(mww_t *h, const int32_t *d_ids, int n, cudaStream_t st) {
    if (n <= 0) return MWW_OK;
    int rc = fill_by_id(h, h->d_carry, kWindow * sizeof(int16_t), d_ids, n, h->n_streams, st);
    if (rc == MWW_OK) rc = fill_by_id(h, h->d_estimate, kNumChannels * sizeof(uint32_t), d_ids, n, h->n_streams, st);
    if (rc == MWW_OK && h->d_rs_hist) rc = fill_by_id(h, h->d_rs_hist, (size_t)h->rs_hist_stride * sizeof(int16_t), d_ids, n, h->n_streams, st);
    if (rc == MWW_OK && h->d_hist) rc = fill_by_id(h, h->d_hist, (size_t)h->hist_cap * sizeof(int16_t), d_ids, n, h->n_streams, st);
    for (size_t k = 0; rc == MWW_OK && k < h->models.size(); ++k) {
        Model &m = h->models[k];
        if (m.members() == h->n_streams) {
            rc = reset_nn_by_id(h, m, m.d_nn_state, m.d_pend, d_ids, n, h->n_streams, st);
            continue;
        }
        if (m.members() == 0) continue;
        if (int rc2 = ensure_ids(h, &h->d_cids, &h->cids_cap, n, st)) return rc2;
        CU(h, launch_compact_ids(h->d_cids, d_ids, n, m.mem.d_inv, h->n_streams, h->sm_count, st));
        h->launches += 1;
        rc = reset_nn_by_id(h, m, m.d_nn_state, m.d_pend, h->d_cids, n, m.members(), st);
    }
    return rc;
}

}  // namespace

int mww_reset(mww_t *h, const int32_t *h_ids, int n, void *cu_stream) {
    if (!h) return MWW_EINVAL;
    ENTER(h);
    cudaStream_t st = static_cast<cudaStream_t>(cu_stream);
    if (!h_ids) {
        if (h->poisoned) {          // whatever the failed staged call left in flight is gone before the state is rebuilt
            cudaDeviceSynchronize();
            h->poisoned = false;
        }
        return zero_state(h, st);
    }
    if (h->poisoned) return fail(h, MWW_ECUDA, "handle needs mww_reset(h, NULL, 0, stream) after a failed staged call");
    if (n <= 0) return MWW_OK;
    for (int i = 0; i < n; ++i)
        if (h_ids[i] < 0 || h_ids[i] >= h->n_streams) return fail(h, MWW_EINVAL, "mww_reset: stream id out of range");
    if (int rc = upload_ids(h, h_ids, n, st)) return rc;
    return reset_by_id(h, h->d_ids, n, st);
}

int mww_reset_device_ids(mww_t *h, const int32_t *d_ids, int n, void *cu_stream) {
    if (!h || (n > 0 && !d_ids) || n < 0) return MWW_EINVAL;
    ENTER_STATEFUL(h);
    return reset_by_id(h, d_ids, n, static_cast<cudaStream_t>(cu_stream));
}

int mww_set_window_step(mww_t *h, int hop_samples) {
    if (!h) return MWW_EINVAL;
    if (hop_samples < 16 || hop_samples > kWindow || (hop_samples & 1))
        return fail(h, MWW_EUNSUPPORTED, "mww_set_window_step: the hop must be an even number of samples in [16, 480] (window_step 1 .. 30 ms)");
    if (h->used != 0) return fail(h, MWW_EINVAL, "mww_set_window_step: the frontend holds buffered samples; reset it first");
    h->hop = hop_samples;
    return MWW_OK;
}

int mww_reset_frontend(mww_t *h, void *cu_stream) {
    if (!h) return MWW_EINVAL;
    ENTER_STATEFUL(h);
    return zero_frontend(h, static_cast<cudaStream_t>(cu_stream));
}

int mww_resample_taps(int rate, int32_t *out, int max_taps, int *n_taps, int *L, int *M) {
    ResamplePlan P;
    if (!resample_plan(rate, &P)) { g_create_error = "mww_resample_taps: unsupported input rate"; return MWW_EUNSUPPORTED; }
    if (n_taps) *n_taps = P.n_taps;
    if (L) *L = P.L;
    if (M) *M = P.M;
    if (!out || max_taps < P.n_taps) return MWW_OK;
    if (!resample_taps(P, out)) { g_create_error = "mww_resample_taps: a phase breaks the partial-sum bound"; return MWW_EINVAL; }
    return MWW_OK;
}

int mww_set_input_rate(mww_t *h, int rate) {
    if (!h) return MWW_EINVAL;
    ResamplePlan P;
    if (!resample_plan(rate, &P))
        return fail(h, MWW_EUNSUPPORTED, "mww_set_input_rate: the input rate must be one of 8000, 16000, 22050, 24000, 32000, 44100, 48000 Hz");
    if (h->used != 0 || h->rs_seen != 0)
        return fail(h, MWW_EINVAL, "mww_set_input_rate: the frontend holds buffered samples; reset it first");
    ENTER_STATEFUL(h);
    int16_t *table = nullptr, *hist = nullptr;
    const int hist_stride = (P.H + 1) / 2 * 2;
    if (P.n_taps > 0) {
        std::vector<int32_t> taps((size_t)P.n_taps);
        if (!resample_taps(P, taps.data())) return fail(h, MWW_EINVAL, "mww_set_input_rate: a phase breaks the partial-sum bound");
        std::vector<int16_t> host((size_t)P.L * P.pitch);
        resample_table(P, taps.data(), host.data());
        const size_t hist_bytes = (size_t)h->n_streams * hist_stride * sizeof(int16_t);
        cudaError_t e = cudaMalloc(&table, host.size() * sizeof(int16_t));
        if (e == cudaSuccess) e = cudaMalloc(&hist, hist_bytes);
        if (e == cudaSuccess) e = cudaMemcpy(table, host.data(), host.size() * sizeof(int16_t), cudaMemcpyHostToDevice);
        if (e == cudaSuccess) e = cudaMemset(hist, 0, hist_bytes);
        if (e != cudaSuccess) {
            cudaFree(table); cudaFree(hist);
            return fail(h, e == cudaErrorMemoryAllocation ? MWW_ENOMEM : MWW_ECUDA, std::string("mww_set_input_rate: ") + cudaGetErrorString(e));
        }
    }
    // earlier calls may still read the old tables, history and member lists
    if (h->d_rs_table || h->d_rs_hist) CU(h, cudaDeviceSynchronize());
    cudaFree(h->d_rs_table); cudaFree(h->d_rs_hist);
    if (h->per_rate) {                 // back to one rate for every stream
        for (RateGroup &g : h->groups) cudaFree(g.d_table);
        cudaFree(h->d_rate_ids); cudaFree(h->d_stream_format);
        for (RateGroup &g : h->groups) g = RateGroup{};
        h->d_rate_ids = nullptr; h->d_stream_format = nullptr;
        h->rate_ids.clear(); h->stream_rate.clear(); h->stream_format.clear();
        for (unsigned &m : h->rate_formats) m = 0;
        h->per_rate = false;
    }
    h->d_rs_table = table; h->d_rs_hist = hist;
    h->rs_hist_stride = P.n_taps > 0 ? hist_stride : 0;
    h->rs = P;
    h->rs_seen = 0;
    return MWW_OK;
}

int mww_get_input_rate(const mww_t *h, int *rate, long long *inputs_seen) {
    if (!h) return MWW_EINVAL;
    if (rate) *rate = h->per_rate ? MWW_RATE_PER_STREAM : h->rs.rate;
    if (inputs_seen) *inputs_seen = h->rs_seen;
    return MWW_OK;
}

int mww_get_resampler_state(mww_t *h, int16_t *h_history, long long *inputs_seen) {
    if (!h) return MWW_EINVAL;
    ENTER_STATEFUL(h);
    if (inputs_seen) *inputs_seen = h->rs_seen;
    if (!h_history || !resampling(h)) return MWW_OK;
    CU(h, cudaDeviceSynchronize());
    const size_t H = (size_t)hist_len(h);
    CU(h, cudaMemcpy2D(h_history, H * 2, h->d_rs_hist, (size_t)h->rs_hist_stride * 2, H * 2, h->n_streams, cudaMemcpyDeviceToHost));
    return MWW_OK;
}

int mww_set_resampler_state(mww_t *h, const int16_t *h_history, long long inputs_seen) {
    if (!h) return MWW_EINVAL;
    if (inputs_seen < 0 || (!resampling(h) && inputs_seen != 0) || (h->per_rate && (inputs_seen & 1)))
        return fail(h, MWW_EINVAL, "mww_set_resampler_state: inputs_seen out of range (always 0 at 16 kHz, even with per-stream rates)");
    ENTER(h);
    CU(h, cudaDeviceSynchronize());
    if (h_history && resampling(h)) {
        const size_t H = (size_t)hist_len(h);
        CU(h, cudaMemcpy2D(h->d_rs_hist, (size_t)h->rs_hist_stride * 2, h_history, H * 2, H * 2, h->n_streams, cudaMemcpyHostToDevice));
    }
    h->rs_seen = inputs_seen;
    return MWW_OK;
}

namespace {

int rate_slot(int rate) {
    for (int i = 0; i < kNumRates; ++i)
        if (kResampleRates[i] == rate) return i;
    return -1;
}

// every group's member list from stream_rate, on the host; the device copy is the caller's
void plan_rate_groups(mww_t *h) {
    h->rate_ids.clear();
    for (RateGroup &g : h->groups) {
        g.off = (int)h->rate_ids.size();
        for (int s = 0; s < h->n_streams; ++s)
            if (h->stream_rate[s] == g.P.rate) h->rate_ids.push_back(s);
        g.n = (int)h->rate_ids.size() - g.off;
    }
}
// the formats present at each rate, from stream_rate and stream_format
void plan_rate_formats(mww_t *h) {
    for (int i = 0; i < kNumRates; ++i) {
        const RateGroup &g = h->groups[i];
        h->rate_formats[i] = 0;
        for (int k = g.off; k < g.off + g.n; ++k) h->rate_formats[i] |= 1u << h->stream_format[(size_t)h->rate_ids[(size_t)k]];
    }
}

// the first mww_set_stream_rates: every rate's table, the [n_streams][H_max] history (zero) and the member list, all streams
// at 16 kHz.  Nothing of the handle changes unless all of it could be allocated.
int enter_per_rate(mww_t *h) {
    RateGroup g[kNumRates];
    const int stride = (resample_max_history() + 1) / 2 * 2;
    int16_t *hist = nullptr;
    int32_t *ids = nullptr;
    uint8_t *formats = nullptr;
    const size_t S = (size_t)h->n_streams;
    cudaError_t e = cudaMalloc(&hist, S * stride * sizeof(int16_t));
    if (e == cudaSuccess) e = cudaMemset(hist, 0, S * stride * sizeof(int16_t));
    if (e == cudaSuccess) e = cudaMalloc(&ids, S * sizeof(int32_t));
    if (e == cudaSuccess) e = cudaMalloc(&formats, S);                  // every stream starts as int16 (kFormatS16 = 0)
    if (e == cudaSuccess) e = cudaMemset(formats, 0, S);
    bool bound = true;
    for (int i = 0; i < kNumRates && e == cudaSuccess && bound; ++i) {
        resample_plan(kResampleRates[i], &g[i].P);
        if (g[i].P.n_taps == 0) continue;
        std::vector<int32_t> taps((size_t)g[i].P.n_taps);
        bound = resample_taps(g[i].P, taps.data());
        std::vector<int16_t> host((size_t)g[i].P.L * g[i].P.pitch);
        resample_table(g[i].P, taps.data(), host.data());
        e = cudaMalloc(&g[i].d_table, host.size() * sizeof(int16_t));
        if (e == cudaSuccess) e = cudaMemcpy(g[i].d_table, host.data(), host.size() * sizeof(int16_t), cudaMemcpyHostToDevice);
    }
    if (e != cudaSuccess || !bound) {
        cudaFree(hist); cudaFree(ids); cudaFree(formats);
        for (RateGroup &r : g) cudaFree(r.d_table);
        if (!bound) return fail(h, MWW_EINVAL, "mww_set_stream_rates: a phase breaks the partial-sum bound");
        return fail(h, e == cudaErrorMemoryAllocation ? MWW_ENOMEM : MWW_ECUDA, std::string("mww_set_stream_rates: ") + cudaGetErrorString(e));
    }
    h->stream_rate.assign(S, 16000);
    h->stream_format.assign(S, kFormatS16);
    for (int i = 0; i < kNumRates; ++i) h->groups[i] = g[i];
    plan_rate_groups(h);
    plan_rate_formats(h);
    if ((e = cudaMemcpy(ids, h->rate_ids.data(), S * sizeof(int32_t), cudaMemcpyHostToDevice)) != cudaSuccess) {
        cudaFree(hist); cudaFree(ids); cudaFree(formats);
        for (RateGroup &r : h->groups) { cudaFree(r.d_table); r = RateGroup{}; }
        h->stream_rate.clear(); h->rate_ids.clear(); h->stream_format.clear();
        for (unsigned &m : h->rate_formats) m = 0;
        return cuda_fail(h, e, "mww_set_stream_rates");
    }
    h->d_rs_hist = hist;
    h->rs_hist_stride = stride;
    h->d_rate_ids = ids;
    h->d_stream_format = formats;
    h->per_rate = true;
    return MWW_OK;
}

}  // namespace

int mww_set_stream_rates(mww_t *h, const int32_t *h_ids, const int32_t *h_rates, int n, void *cu_stream) {
    if (!h) return MWW_EINVAL;
    if (n < 0 || (n > 0 && (!h_ids || !h_rates))) return fail(h, MWW_EINVAL, "mww_set_stream_rates: bad arguments");
    std::vector<char> listed((size_t)h->n_streams, 0);
    for (int i = 0; i < n; ++i) {
        if (h_ids[i] < 0 || h_ids[i] >= h->n_streams) return fail(h, MWW_EINVAL, "mww_set_stream_rates: stream id out of range");
        if (listed[(size_t)h_ids[i]]) return fail(h, MWW_EINVAL, "mww_set_stream_rates: duplicate stream id");
        listed[(size_t)h_ids[i]] = 1;
    }
    for (int i = 0; i < n; ++i)
        if (rate_slot(h_rates[i]) < 0)
            return fail(h, MWW_EUNSUPPORTED, "mww_set_stream_rates: every rate must be one of 8000, 16000, 22050, 24000, 32000, 44100, 48000 Hz");
    if (!h->per_rate && (h->used != 0 || h->rs_seen != 0 || h->rs.rate != 16000))
        return fail(h, MWW_EINVAL, "mww_set_stream_rates: per-stream rates start on a 16 kHz handle that holds no buffered samples; reset it first");
    ENTER_STATEFUL(h);
    cudaStream_t st = static_cast<cudaStream_t>(cu_stream);
    if (!h->per_rate)
        if (int rc = enter_per_rate(h)) return rc;
    if (n == 0) return MWW_OK;
    // the listed streams' histories are zeroed, then the member lists change, both in stream order
    if (int rc = upload_ids(h, h_ids, n, st)) return rc;
    if (int rc = fill_by_id(h, h->d_rs_hist, (size_t)h->rs_hist_stride * sizeof(int16_t), h->d_ids, n, h->n_streams, st)) return rc;
    for (int i = 0; i < n; ++i) h->stream_rate[(size_t)h_ids[i]] = h_rates[i];
    plan_rate_groups(h);
    plan_rate_formats(h);
    CU(h, cudaMemcpyAsync(h->d_rate_ids, h->rate_ids.data(), (size_t)h->n_streams * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    return MWW_OK;
}

int mww_get_stream_rates(const mww_t *h, int32_t *h_rates, long long *samples16_seen) {
    if (!h) return MWW_EINVAL;
    if (h_rates)
        for (int s = 0; s < h->n_streams; ++s) h_rates[s] = h->per_rate ? h->stream_rate[(size_t)s] : h->rs.rate;
    if (samples16_seen) *samples16_seen = h->per_rate ? h->rs_seen : resample_outputs(h->rs_seen, h->rs.L, h->rs.M);
    return MWW_OK;
}

int mww_rate_inputs(int rate, long long samples16, long long *inputs) {
    ResamplePlan P;
    if (!resample_plan(rate, &P)) { g_create_error = "mww_rate_inputs: unsupported input rate"; return MWW_EUNSUPPORTED; }
    if (samples16 < 0 || samples16 > (1ll << 50) || !inputs) { g_create_error = "mww_rate_inputs: bad arguments"; return MWW_EINVAL; }
    *inputs = resample_inputs(samples16, P.L, P.M);
    return MWW_OK;
}

static_assert(kFormatS16 == MWW_FORMAT_S16 && kFormatUlaw == MWW_FORMAT_ULAW && kFormatAlaw == MWW_FORMAT_ALAW && kFormatF32 == MWW_FORMAT_F32 &&
              MWW_FORMAT_ULAW == MWW_G711_ULAW && MWW_FORMAT_ALAW == MWW_G711_ALAW, "format codes");

int mww_set_stream_formats(mww_t *h, const int32_t *h_ids, const int32_t *h_formats, int n, void *cu_stream) {
    if (!h) return MWW_EINVAL;
    if (!h->per_rate)
        return fail(h, MWW_EUNSUPPORTED, "mww_set_stream_formats: sample formats per stream need per-stream rates (mww_set_stream_rates)");
    if (n < 0 || (n > 0 && (!h_ids || !h_formats))) return fail(h, MWW_EINVAL, "mww_set_stream_formats: bad arguments");
    std::vector<char> listed((size_t)h->n_streams, 0);
    for (int i = 0; i < n; ++i) {
        if (h_ids[i] < 0 || h_ids[i] >= h->n_streams) return fail(h, MWW_EINVAL, "mww_set_stream_formats: stream id out of range");
        if (listed[(size_t)h_ids[i]]) return fail(h, MWW_EINVAL, "mww_set_stream_formats: duplicate stream id");
        listed[(size_t)h_ids[i]] = 1;
        if (h_formats[i] < 0 || h_formats[i] >= kNumFormats)
            return fail(h, MWW_EINVAL, "mww_set_stream_formats: a format must be MWW_FORMAT_S16, _ULAW, _ALAW or _F32, not " + std::to_string(h_formats[i]));
    }
    ENTER_STATEFUL(h);
    if (n == 0) return MWW_OK;
    std::vector<uint8_t> next = h->stream_format;
    for (int i = 0; i < n; ++i) next[(size_t)h_ids[i]] = (uint8_t)h_formats[i];
    // pageable source: the copy has taken the bytes when it returns
    CU(h, cudaMemcpyAsync(h->d_stream_format, next.data(), next.size(), cudaMemcpyHostToDevice, static_cast<cudaStream_t>(cu_stream)));
    h->stream_format.swap(next);
    plan_rate_formats(h);
    return MWW_OK;
}

int mww_get_stream_formats(const mww_t *h, int32_t *h_formats) {
    if (!h || !h_formats) return MWW_EINVAL;
    for (int s = 0; s < h->n_streams; ++s) h_formats[s] = h->per_rate ? h->stream_format[(size_t)s] : kFormatS16;
    return MWW_OK;
}

int mww_features(mww_t *h, const int16_t *d_audio, int n_samples, long long audio_stride, uint16_t *d_feat, int max_rows,
                 int *h_rows_out, void *cu_stream) {
    return features_impl(h, "mww_features", d_audio, n_samples, audio_stride, d_feat, max_rows, h_rows_out, cu_stream);
}
int mww_features_f32(mww_t *h, const float *d_audio, int n_samples, long long audio_stride, uint16_t *d_feat, int max_rows,
                     int *h_rows_out, void *cu_stream) {
    return features_impl(h, "mww_features_f32", d_audio, n_samples, audio_stride, d_feat, max_rows, h_rows_out, cu_stream);
}

int mww_predict_clip(mww_t *h, const int16_t *d_audio, int n_samples, long long audio_stride, float *d_probs, int max_probs,
                     int *h_probs_out, void *cu_stream) {
    if (int rc = refuse_multi(h, "mww_predict_clip", "mww_predict_clip_multi")) return rc;
    return predict_clip_impl(h, "mww_predict_clip", d_audio, n_samples, audio_stride, &d_probs, &max_probs, h_probs_out, cu_stream);
}
int mww_predict_clip_f32(mww_t *h, const float *d_audio, int n_samples, long long audio_stride, float *d_probs, int max_probs,
                         int *h_probs_out, void *cu_stream) {
    if (int rc = refuse_multi(h, "mww_predict_clip_f32", "mww_predict_clip_multi_f32")) return rc;
    return predict_clip_impl(h, "mww_predict_clip_f32", d_audio, n_samples, audio_stride, &d_probs, &max_probs, h_probs_out, cu_stream);
}
int mww_predict_clip_multi(mww_t *h, const int16_t *d_audio, int n_samples, long long audio_stride, float *const *d_probs,
                           const int *max_probs, int *h_probs_out, void *cu_stream) {
    return predict_clip_impl(h, "mww_predict_clip_multi", d_audio, n_samples, audio_stride, d_probs, max_probs, h_probs_out, cu_stream);
}
int mww_predict_clip_multi_f32(mww_t *h, const float *d_audio, int n_samples, long long audio_stride, float *const *d_probs,
                               const int *max_probs, int *h_probs_out, void *cu_stream) {
    return predict_clip_impl(h, "mww_predict_clip_multi_f32", d_audio, n_samples, audio_stride, d_probs, max_probs, h_probs_out, cu_stream);
}

int mww_infer_features(mww_t *h, const void *d_rows, int row_type, int n_rows, long long rows_stride, float *d_probs,
                       int max_probs, int *h_probs_out, void *cu_stream) {
    if (!h) return MWW_EINVAL;
    if (int rc = refuse_multi(h, "mww_infer_features", "mww_predict_clip_multi")) return rc;
    if (n_rows < 0 || (n_rows > 0 && !d_rows) || rows_stride < n_rows) return fail(h, MWW_EINVAL, "mww_infer_features: bad row arguments");
    if (row_type < 0 || row_type > 2) return fail(h, MWW_EINVAL, "mww_infer_features: unknown row_type");
    if (h->models.empty()) return fail(h, MWW_EINVAL, "mww_infer_features: frontend-only handle (created without a model)");
    ENTER_STATEFUL(h);
    Model &m = h->models[0];
    const int n_steps = (m.n_pend + n_rows) / m.G.stride;
    if (n_steps > max_probs || (n_steps > 0 && !d_probs)) return fail(h, MWW_EINVAL, "mww_infer_features: probability buffer too small");
    int rc = begin_nn_call(h, m, n_rows, static_cast<cudaStream_t>(cu_stream));
    if (rc) return rc;
    m.tc_rows_bounded = false;          // the caller's rows may hold any value, and the state will carry them
    rc = run_nn_tile(h, m, 0, h->n_streams, d_rows, row_type, rows_stride, n_rows, d_probs, max_probs, static_cast<cudaStream_t>(cu_stream));
    if (rc == MWW_OK) end_nn_call(h, m, n_rows);
    if (rc) return rc;
    m.n_pend = (m.n_pend + n_rows) % m.G.stride;
    if (h_probs_out) *h_probs_out = n_steps;
    return MWW_OK;
}

// ---- staged path: the audio does not live on this GPU ------------------------------------------------------------
// Shared by mww_predict_clip_host (source = host memory, destination = host memory) and mww_predict_clip_remote (source =
// host memory or device memory of a PEER GPU mapped into this process, destination = this GPU).  The streams are cut into
// tiles; a copy stream brings tile t+1 into one of two staging buffers (cudaMemcpyAsync, cudaMemcpyDefault: the copy
// engine of THIS GPU pulls over PCIe or NVLink, no SM is involved on either side) while the kernels of tile t run on the
// compute stream, and for a host destination a third stream drains the scores.  The bodies are templates over the sample
// type (int16_t, float, or the G.711 types), hence C++ linkage.
extern "C++" {
namespace {

int ensure_pipeline(mww_t *h) {
    if (h->st_compute) return MWW_OK;
    CU(h, cudaStreamCreateWithFlags(&h->st_h2d, cudaStreamNonBlocking));
    CU(h, cudaStreamCreateWithFlags(&h->st_compute, cudaStreamNonBlocking));
    CU(h, cudaStreamCreateWithFlags(&h->st_d2h, cudaStreamNonBlocking));
    for (int b = 0; b < 2; ++b) {
        CU(h, cudaEventCreateWithFlags(&h->ev_h2d[b], cudaEventDisableTiming));
        CU(h, cudaEventCreateWithFlags(&h->ev_compute[b], cudaEventDisableTiming));
        CU(h, cudaEventCreateWithFlags(&h->ev_d2h[b], cudaEventDisableTiming));
    }
    CU(h, cudaEventCreateWithFlags(&h->ev_entry, cudaEventDisableTiming));
    CU(h, cudaEventCreateWithFlags(&h->ev_exit, cudaEventDisableTiming));
    return MWW_OK;
}

// the tile loop proper; any error leaves work in flight -- the caller drains the streams and poisons the handle
// Model k's scores of a tile go to dst[k] at its stream pitch; for a host destination they are first written to the score
// staging buffer, where model k's block of tile x max(steps, 1) floats starts at probs_tile_offset(o, tile, k).
size_t probs_tile_offset(const mww_t *h, const NnOuts &o, int tile, size_t k) {
    size_t off = 0;
    for (size_t j = 0; j < k && j < h->models.size(); ++j) off += (size_t)tile * std::max(o.steps[j], 1);
    return off;
}

// T = int16_t, float, Ulaw8 or Alaw8: the staging buffers hold the caller's samples as they are, and the frontend and carry
// kernels of that sample type convert them (as on the device path); Mixed8: the bytes of mixed rows, which the resampler
// decodes
template <typename T>
int staged_tiles(mww_t *h, const T *src, int n_samples, long long audio_stride, const NnOuts &o, bool dst_is_host,
                 int tile, int n_frames, int n16) {
    const size_t K = h->models.size();
    const T *audio_tile[2] = {static_cast<const T *>(h->d_audio_tile[0]), static_cast<const T *>(h->d_audio_tile[1])};
    const long long call_width = row_width<T>(h, n_samples);      // samples per staged row
    float *tile_probs[kMaxModels];
    long long tile_probs_stride[kMaxModels];
    TileSpan span[kMaxModels];
    for (size_t k = 0; k < K; ++k) tile_probs_stride[k] = dst_is_host ? std::max(o.steps[k], 1) : o.max_probs[k];
    int it = 0;
    for (int first = 0; first < h->n_streams; first += tile, ++it) {
        const int n = std::min(tile, h->n_streams - first);
        const int b = it & 1;
        // mixed rows: as many bytes as the tile's widest row, rounded up to 4 so that its float rows stay aligned
        long long width = call_width;
        if constexpr (std::is_same<T, Mixed8>::value) width = (mixed_tile_width(h, first, n, n_samples) + 3) / 4 * 4;
        // the staging buffer is free once the kernels of the tile that used it two iterations ago are done
        if (it >= 2) CU(h, cudaStreamWaitEvent(h->st_h2d, h->ev_compute[b], 0));
        cudaEvent_t tl[4] = {nullptr, nullptr, nullptr, nullptr};
        if (h->profiling) {
            for (int i = 0; i < 4; ++i) { CU(h, cudaEventCreate(&tl[i])); h->tl_ev.push_back(tl[i]); }
            CU(h, cudaEventRecord(tl[0], h->st_h2d));
        }
        if (width > 0) {
            const T *from = src + (size_t)first * audio_stride;
            const size_t row = (size_t)width * sizeof(T);
            if (audio_stride == width)           // contiguous block: one linear DMA
                CU(h, cudaMemcpyAsync(h->d_audio_tile[b], from, (size_t)n * row, cudaMemcpyDefault, h->st_h2d));
            else
                CU(h, cudaMemcpy2DAsync(h->d_audio_tile[b], row, from, (size_t)audio_stride * sizeof(T), row, n,
                                        cudaMemcpyDefault, h->st_h2d));
        }
        if (tl[1]) CU(h, cudaEventRecord(tl[1], h->st_h2d));
        CU(h, cudaEventRecord(h->ev_h2d[b], h->st_h2d));
        CU(h, cudaStreamWaitEvent(h->st_compute, h->ev_h2d[b], 0));
        if (tl[2]) CU(h, cudaEventRecord(tl[2], h->st_compute));
        if (dst_is_host && it >= 2) CU(h, cudaStreamWaitEvent(h->st_compute, h->ev_d2h[b], 0));   // score staging buffer drained
        int rc = MWW_OK;
        if (resampling(h)) {
            // one 16 kHz scratch serves every tile: all kernels run in order on the compute stream
            rc = run_resample_tile(h, first, n, audio_tile[b], width, n_samples, n16, h->st_compute);
            if (rc == MWW_OK) rc = run_frontend_tile(h, first, n, h->d_rs_out, n16, n16, n_frames, h->d_feat, (long long)n_frames * kNumChannels, h->st_compute);
        } else {
            rc = run_frontend_tile(h, first, n, audio_tile[b], n_samples, n_samples, n_frames, h->d_feat, (long long)n_frames * kNumChannels, h->st_compute);
        }
        if (rc) return rc;
        tile_spans(h, first, n, span);
        for (size_t k = 0; k < K; ++k)
            tile_probs[k] = dst_is_host ? h->d_probs_tile[b] + probs_tile_offset(h, o, tile, k) : o.probs[k] + (size_t)span[k].a * o.max_probs[k];
        rc = run_models_tile(h, first, n_frames, span, tile_probs, tile_probs_stride, h->st_compute);
        if (rc) return rc;
        if (resampling(h) ? n16 > 0 : n_samples > 0) {
            rc = resampling(h) ? run_carry_tile(h, first, n, h->d_rs_out, n16, n16, n_frames, h->st_compute)
                               : run_carry_tile(h, first, n, audio_tile[b], n_samples, n_samples, n_frames, h->st_compute);
            if (rc) return rc;
        }
        rc = resampling(h) ? run_history_tile(h, first, n, h->d_rs_out, n16, n16, h->st_compute)
                           : run_history_tile(h, first, n, audio_tile[b], n_samples, n_samples, h->st_compute);
        if (rc) return rc;
        if (tl[3]) CU(h, cudaEventRecord(tl[3], h->st_compute));
        CU(h, cudaEventRecord(h->ev_compute[b], h->st_compute));
        if (dst_is_host) {
            CU(h, cudaStreamWaitEvent(h->st_d2h, h->ev_compute[b], 0));
            for (size_t k = 0; k < K; ++k)
                if (o.steps[k] > 0 && span[k].b > span[k].a)      // model k's rows [a, b) of the tile
                    CU(h, cudaMemcpy2DAsync(o.probs[k] + (size_t)span[k].a * o.max_probs[k], (size_t)o.max_probs[k] * 4, tile_probs[k],
                                            (size_t)tile_probs_stride[k] * 4, (size_t)o.steps[k] * 4, span[k].b - span[k].a,
                                            cudaMemcpyDeviceToHost, h->st_d2h));
            CU(h, cudaEventRecord(h->ev_d2h[b], h->st_d2h));
        }
    }
    return MWW_OK;
}

// `caller` != nullptr-or-legacy semantics: the call is ordered after everything queued on `caller` so far, and `caller`
// is made to wait for the call's last kernel (asynchronous variant).  host_sync: return only when dst is complete.
template <typename T>
int predict_clip_staged(mww_t *h, const char *who, const T *src, int n_samples, long long audio_stride, float *const *dst,
                        const int *max_probs, int *h_probs_out, bool dst_is_host, int want_tiles, cudaStream_t caller, bool host_sync) {
    if (!resample_call_fits(h, n_samples)) return fail(h, MWW_EINVAL, std::string(who) + ": call too long for the resampler; split it");
    const int n16 = samples16(h, n_samples);
    const int n_frames = frames_for(h, n16);
    NnOuts o;
    int rc = check_outs(h, who, n_frames, dst, max_probs, &o);
    if (rc) return rc;
    rc = ensure_pipeline(h);
    if (rc) return rc;
    // tile so that copies and kernels of neighbouring tiles overlap: 16 tiles by default when there are enough streams (the
    // first tile's copy and the last tile's kernels are the only parts that cannot hide behind each other), but never
    // fewer than 2 048 streams per tile so that every launch still fills the GPU
    if (want_tiles <= 0) want_tiles = 16;
    // float32 samples double the staging buffers, so their two tiles count against the scratch budget (MWW_SCRATCH_MB) with
    // the scratch; int16 tiles keep the sizing they have always had, from the scratch alone, and G.711 tiles (half an int16
    // tile) need nothing beyond that either.  A resampling handle adds its 16 kHz tile scratch.  Mixed rows count their two
    // tiles at the call's widest row in bytes, rounded up to 4 as each tile's rows are.
    constexpr bool mixed = std::is_same<T, Mixed8>::value;
    long long width = row_width<T>(h, n_samples);      // per-stream rates: the call's largest D_s (mixed rows: bytes)
    if (mixed) width = (width + 3) / 4 * 4;
    const size_t staged_bytes = sizeof(T) <= sizeof(int16_t) && !mixed ? 0 : 2 * (size_t)std::max<long long>(width, 1) * sizeof(T);
    const size_t gather = gather_bytes_per_stream(h, n_frames);
    int tile = tile_streams(h, n_frames, true, staged_bytes + gather + (resampling(h) ? (size_t)n16 * 2 : 0));
    tile = std::max(1, std::min(tile, std::max((h->n_streams + want_tiles - 1) / want_tiles, std::min(h->n_streams, h->min_tile_streams))));
    rc = ensure_scratch(h, v_scratch_bytes(h, tile, n_frames), (size_t)tile * std::max(n_frames, 1) * kNumChannels * 2, (size_t)tile * gather);
    if (rc == MWW_OK && resampling(h)) rc = ensure_rs_out(h, (size_t)tile * std::max(n16, 1) * 2);
    if (rc) return rc;
    const size_t a_bytes = (size_t)tile * std::max<long long>(width, 1) * sizeof(T);
    const size_t p_bytes = dst_is_host ? probs_tile_offset(h, o, tile, h->models.size()) * sizeof(float) : 0;
    if (a_bytes > h->audio_tile_bytes || p_bytes > h->probs_tile_bytes) {
        CU(h, cudaDeviceSynchronize());
        for (int b = 0; b < 2; ++b) {
            cudaFree(h->d_audio_tile[b]); cudaFree(h->d_probs_tile[b]);
            h->d_audio_tile[b] = nullptr; h->d_probs_tile[b] = nullptr;
        }
        const size_t a_new = std::max(a_bytes, h->audio_tile_bytes), p_new = std::max(p_bytes, h->probs_tile_bytes);
        h->audio_tile_bytes = h->probs_tile_bytes = 0;
        for (int b = 0; b < 2; ++b) {
            CU(h, cudaMalloc(&h->d_audio_tile[b], a_new));
            if (p_new) CU(h, cudaMalloc(&h->d_probs_tile[b], p_new));
        }
        h->audio_tile_bytes = a_new; h->probs_tile_bytes = p_new;
    }
    // order the private streams after the caller's outstanding work (mww_reset, earlier live calls, the producer of a
    // device-resident source) and after whatever an earlier staged call still has in flight on the staging buffers
    CU(h, cudaEventRecord(h->ev_entry, caller));
    CU(h, cudaStreamWaitEvent(h->st_h2d, h->ev_entry, 0));
    CU(h, cudaStreamWaitEvent(h->st_compute, h->ev_entry, 0));
    if (h->staged_used)
        for (int b = 0; b < 2; ++b) CU(h, cudaStreamWaitEvent(h->st_h2d, h->ev_compute[b], 0));
    for (cudaEvent_t e : h->tl_ev) cudaEventDestroy(e);       // a timeline describes the most recent staged call only
    h->tl_ev.clear();
    rc = begin_models_call(h, n_frames, h->st_compute);
    if (rc == MWW_OK) {
        h->staged_used = true;
        rc = staged_tiles(h, src, n_samples, audio_stride, o, dst_is_host, tile, n_frames, n16);
    }
    if (rc != MWW_OK) {
        // some tiles' carry / ring state may already be updated, others not: drain and refuse further stateful calls
        const std::string msg = h->err;
        cudaStreamSynchronize(h->st_h2d); cudaStreamSynchronize(h->st_compute); cudaStreamSynchronize(h->st_d2h);
        h->poisoned = true;
        h->err = msg + " (staged call aborted; mww_reset(h, NULL, 0, stream) required)";
        return rc;
    }
    if (host_sync) {
        CU(h, cudaStreamSynchronize(h->st_d2h));
        CU(h, cudaStreamSynchronize(h->st_compute));
    } else {
        CU(h, cudaEventRecord(h->ev_exit, h->st_compute));
        CU(h, cudaStreamWaitEvent(caller, h->ev_exit, 0));
    }
    end_models_call(h, n_frames, o, h_probs_out);
    h->used = h->used + n16 - n_frames * h->hop;
    if (resampling(h)) h->rs_seen += n_samples;
    end_history_call(h, n16);
    return MWW_OK;
}

template <typename T>
int predict_clip_host_impl(mww_t *h, const char *who, const T *h_audio, int n_samples, long long audio_stride, float *const *h_probs,
                           const int *max_probs, int *h_probs_out) {
    if (!h) return MWW_EINVAL;
    if (bad_audio(h, n_samples, h_audio, audio_stride)) return fail(h, MWW_EINVAL, std::string(who) + ": bad audio arguments");
    if (h->models.empty()) return fail(h, MWW_EINVAL, std::string(who) + ": frontend-only handle (created without a model)");
    ENTER_STATEFUL(h);
    // The call has no stream argument, so it cannot be ordered after one particular stream: it waits for everything the
    // device has been given so far (mww_reset / live calls queued on any stream touch the same per-stream state).
    CU(h, cudaDeviceSynchronize());
    return predict_clip_staged(h, who, h_audio, n_samples, audio_stride, h_probs, max_probs, h_probs_out, true, 0, nullptr, true);
}

template <typename T>
int predict_clip_remote_impl(mww_t *h, const char *who, const T *src_audio, int n_samples, long long audio_stride, float *const *d_probs,
                             const int *max_probs, int *h_probs_out, int n_tiles, void *cu_stream) {
    if (!h) return MWW_EINVAL;
    if (bad_audio(h, n_samples, src_audio, audio_stride)) return fail(h, MWW_EINVAL, std::string(who) + ": bad audio arguments");
    if (h->models.empty()) return fail(h, MWW_EINVAL, std::string(who) + ": frontend-only handle (created without a model)");
    bool local = n_samples == 0;
    if (!local) {
        DeviceGuard guard(h->device);
        cudaPointerAttributes at;
        memset(&at, 0, sizeof at);
        if (cudaPointerGetAttributes(&at, src_audio) != cudaSuccess) { cudaGetLastError(); memset(&at, 0, sizeof at); }
        local = (at.type == cudaMemoryTypeDevice && at.device == h->device) || at.type == cudaMemoryTypeManaged;
    }
    // a source this GPU's kernels can address -- its own memory, or a peer's buffer mapped with mww_ipc_open, which reports this
    // device too -- is read in place by the frontend kernel unless the caller asks for the staged pipeline (n_tiles > 0)
    if (local && n_tiles <= 0) return predict_clip_impl(h, who, src_audio, n_samples, audio_stride, d_probs, max_probs, h_probs_out, cu_stream);
    ENTER_STATEFUL(h);
    return predict_clip_staged(h, who, src_audio, n_samples, audio_stride, d_probs, max_probs, h_probs_out, false, n_tiles,
                               static_cast<cudaStream_t>(cu_stream), false);
}

}  // namespace
}  // extern "C++"

int mww_predict_clip_host(mww_t *h, const int16_t *h_audio, int n_samples, long long audio_stride, float *h_probs, int max_probs,
                          int *h_probs_out) {
    if (int rc = refuse_multi(h, "mww_predict_clip_host", "mww_predict_clip_host_multi")) return rc;
    return predict_clip_host_impl(h, "mww_predict_clip_host", h_audio, n_samples, audio_stride, &h_probs, &max_probs, h_probs_out);
}
int mww_predict_clip_host_multi(mww_t *h, const int16_t *h_audio, int n_samples, long long audio_stride, float *const *h_probs,
                                const int *max_probs, int *h_probs_out) {
    return predict_clip_host_impl(h, "mww_predict_clip_host_multi", h_audio, n_samples, audio_stride, h_probs, max_probs, h_probs_out);
}

int mww_predict_clip_remote(mww_t *h, const int16_t *src_audio, int n_samples, long long audio_stride, float *d_probs, int max_probs,
                            int *h_probs_out, int n_tiles, void *cu_stream) {
    if (int rc = refuse_multi(h, "mww_predict_clip_remote", "mww_predict_clip_remote_multi")) return rc;
    return predict_clip_remote_impl(h, "mww_predict_clip_remote", src_audio, n_samples, audio_stride, &d_probs, &max_probs, h_probs_out, n_tiles,
                                    cu_stream);
}
int mww_predict_clip_remote_multi(mww_t *h, const int16_t *src_audio, int n_samples, long long audio_stride, float *const *d_probs,
                                  const int *max_probs, int *h_probs_out, int n_tiles, void *cu_stream) {
    return predict_clip_remote_impl(h, "mww_predict_clip_remote_multi", src_audio, n_samples, audio_stride, d_probs, max_probs, h_probs_out,
                                    n_tiles, cu_stream);
}

int mww_predict_clip_host_f32(mww_t *h, const float *h_audio, int n_samples, long long audio_stride, float *h_probs, int max_probs,
                              int *h_probs_out) {
    if (int rc = refuse_multi(h, "mww_predict_clip_host_f32", "mww_predict_clip_host_multi_f32")) return rc;
    return predict_clip_host_impl(h, "mww_predict_clip_host_f32", h_audio, n_samples, audio_stride, &h_probs, &max_probs, h_probs_out);
}
int mww_predict_clip_host_multi_f32(mww_t *h, const float *h_audio, int n_samples, long long audio_stride, float *const *h_probs,
                                    const int *max_probs, int *h_probs_out) {
    return predict_clip_host_impl(h, "mww_predict_clip_host_multi_f32", h_audio, n_samples, audio_stride, h_probs, max_probs, h_probs_out);
}

int mww_predict_clip_remote_f32(mww_t *h, const float *src_audio, int n_samples, long long audio_stride, float *d_probs, int max_probs,
                                int *h_probs_out, int n_tiles, void *cu_stream) {
    if (int rc = refuse_multi(h, "mww_predict_clip_remote_f32", "mww_predict_clip_remote_multi_f32")) return rc;
    return predict_clip_remote_impl(h, "mww_predict_clip_remote_f32", src_audio, n_samples, audio_stride, &d_probs, &max_probs, h_probs_out,
                                    n_tiles, cu_stream);
}
int mww_predict_clip_remote_multi_f32(mww_t *h, const float *src_audio, int n_samples, long long audio_stride, float *const *d_probs,
                                      const int *max_probs, int *h_probs_out, int n_tiles, void *cu_stream) {
    return predict_clip_remote_impl(h, "mww_predict_clip_remote_multi_f32", src_audio, n_samples, audio_stride, d_probs, max_probs,
                                    h_probs_out, n_tiles, cu_stream);
}

// ---- G.711 audio: the bodies above with the law as the sample type (Ulaw8 / Alaw8, decoded inside the kernels) ----------
extern "C++" {
namespace {

// run(audio as the law's sample type); a law other than the two is refused before anything else looks at the handle's state
template <typename F>
int with_law(mww_t *h, const char *who, int law, const uint8_t *audio, F run) {
    if (!h) return MWW_EINVAL;
    if (law == MWW_G711_ULAW) return run(reinterpret_cast<const Ulaw8 *>(audio));
    if (law == MWW_G711_ALAW) return run(reinterpret_cast<const Alaw8 *>(audio));
    return fail(h, MWW_EINVAL, std::string(who) + ": law must be MWW_G711_ULAW (1) or MWW_G711_ALAW (2), not " + std::to_string(law));
}

// run(audio as mixed rows); a handle without per-stream rates is refused before anything else looks at its state
template <typename F>
int with_mixed(mww_t *h, const char *who, const uint8_t *audio, F run) {
    if (!h) return MWW_EINVAL;
    if (!h->per_rate) return fail(h, MWW_EUNSUPPORTED, std::string(who) + ": mixed rows need per-stream rates (mww_set_stream_rates)");
    return run(reinterpret_cast<const Mixed8 *>(audio));
}

}  // namespace
}  // extern "C++"

int mww_features_g711(mww_t *h, const uint8_t *d_audio, int law, int n_samples, long long audio_stride, uint16_t *d_feat, int max_rows,
                      int *h_rows_out, void *cu_stream) {
    return with_law(h, "mww_features_g711", law, d_audio, [&](auto a) {
        return features_impl(h, "mww_features_g711", a, n_samples, audio_stride, d_feat, max_rows, h_rows_out, cu_stream);
    });
}
int mww_predict_clip_g711(mww_t *h, const uint8_t *d_audio, int law, int n_samples, long long audio_stride, float *d_probs, int max_probs,
                          int *h_probs_out, void *cu_stream) {
    return with_law(h, "mww_predict_clip_g711", law, d_audio, [&](auto a) {
        if (int rc = refuse_multi(h, "mww_predict_clip_g711", "mww_predict_clip_multi_g711")) return rc;
        return predict_clip_impl(h, "mww_predict_clip_g711", a, n_samples, audio_stride, &d_probs, &max_probs, h_probs_out, cu_stream);
    });
}
int mww_predict_clip_multi_g711(mww_t *h, const uint8_t *d_audio, int law, int n_samples, long long audio_stride, float *const *d_probs,
                                const int *max_probs, int *h_probs_out, void *cu_stream) {
    return with_law(h, "mww_predict_clip_multi_g711", law, d_audio, [&](auto a) {
        return predict_clip_impl(h, "mww_predict_clip_multi_g711", a, n_samples, audio_stride, d_probs, max_probs, h_probs_out, cu_stream);
    });
}
int mww_predict_clip_host_g711(mww_t *h, const uint8_t *h_audio, int law, int n_samples, long long audio_stride, float *h_probs,
                               int max_probs, int *h_probs_out) {
    return with_law(h, "mww_predict_clip_host_g711", law, h_audio, [&](auto a) {
        if (int rc = refuse_multi(h, "mww_predict_clip_host_g711", "mww_predict_clip_host_multi_g711")) return rc;
        return predict_clip_host_impl(h, "mww_predict_clip_host_g711", a, n_samples, audio_stride, &h_probs, &max_probs, h_probs_out);
    });
}
int mww_predict_clip_host_multi_g711(mww_t *h, const uint8_t *h_audio, int law, int n_samples, long long audio_stride,
                                     float *const *h_probs, const int *max_probs, int *h_probs_out) {
    return with_law(h, "mww_predict_clip_host_multi_g711", law, h_audio, [&](auto a) {
        return predict_clip_host_impl(h, "mww_predict_clip_host_multi_g711", a, n_samples, audio_stride, h_probs, max_probs, h_probs_out);
    });
}
int mww_predict_clip_remote_g711(mww_t *h, const uint8_t *src_audio, int law, int n_samples, long long audio_stride, float *d_probs,
                                 int max_probs, int *h_probs_out, int n_tiles, void *cu_stream) {
    return with_law(h, "mww_predict_clip_remote_g711", law, src_audio, [&](auto a) {
        if (int rc = refuse_multi(h, "mww_predict_clip_remote_g711", "mww_predict_clip_remote_multi_g711")) return rc;
        return predict_clip_remote_impl(h, "mww_predict_clip_remote_g711", a, n_samples, audio_stride, &d_probs, &max_probs, h_probs_out,
                                        n_tiles, cu_stream);
    });
}
int mww_predict_clip_remote_multi_g711(mww_t *h, const uint8_t *src_audio, int law, int n_samples, long long audio_stride,
                                       float *const *d_probs, const int *max_probs, int *h_probs_out, int n_tiles, void *cu_stream) {
    return with_law(h, "mww_predict_clip_remote_multi_g711", law, src_audio, [&](auto a) {
        return predict_clip_remote_impl(h, "mww_predict_clip_remote_multi_g711", a, n_samples, audio_stride, d_probs, max_probs,
                                        h_probs_out, n_tiles, cu_stream);
    });
}

// ---- mixed rows: the bodies above with a sample format per stream (Mixed8 bytes, decoded by the resampler) --------------
int mww_features_mixed(mww_t *h, const uint8_t *d_audio, int n_samples, long long audio_stride, uint16_t *d_feat, int max_rows,
                       int *h_rows_out, void *cu_stream) {
    return with_mixed(h, "mww_features_mixed", d_audio, [&](auto a) {
        return features_impl(h, "mww_features_mixed", a, n_samples, audio_stride, d_feat, max_rows, h_rows_out, cu_stream);
    });
}
int mww_predict_clip_mixed(mww_t *h, const uint8_t *d_audio, int n_samples, long long audio_stride, float *d_probs, int max_probs,
                           int *h_probs_out, void *cu_stream) {
    return with_mixed(h, "mww_predict_clip_mixed", d_audio, [&](auto a) {
        if (int rc = refuse_multi(h, "mww_predict_clip_mixed", "mww_predict_clip_multi_mixed")) return rc;
        return predict_clip_impl(h, "mww_predict_clip_mixed", a, n_samples, audio_stride, &d_probs, &max_probs, h_probs_out, cu_stream);
    });
}
int mww_predict_clip_multi_mixed(mww_t *h, const uint8_t *d_audio, int n_samples, long long audio_stride, float *const *d_probs,
                                 const int *max_probs, int *h_probs_out, void *cu_stream) {
    return with_mixed(h, "mww_predict_clip_multi_mixed", d_audio, [&](auto a) {
        return predict_clip_impl(h, "mww_predict_clip_multi_mixed", a, n_samples, audio_stride, d_probs, max_probs, h_probs_out, cu_stream);
    });
}
int mww_predict_clip_host_mixed(mww_t *h, const uint8_t *h_audio, int n_samples, long long audio_stride, float *h_probs, int max_probs,
                                int *h_probs_out) {
    return with_mixed(h, "mww_predict_clip_host_mixed", h_audio, [&](auto a) {
        if (int rc = refuse_multi(h, "mww_predict_clip_host_mixed", "mww_predict_clip_host_multi_mixed")) return rc;
        return predict_clip_host_impl(h, "mww_predict_clip_host_mixed", a, n_samples, audio_stride, &h_probs, &max_probs, h_probs_out);
    });
}
int mww_predict_clip_host_multi_mixed(mww_t *h, const uint8_t *h_audio, int n_samples, long long audio_stride, float *const *h_probs,
                                      const int *max_probs, int *h_probs_out) {
    return with_mixed(h, "mww_predict_clip_host_multi_mixed", h_audio, [&](auto a) {
        return predict_clip_host_impl(h, "mww_predict_clip_host_multi_mixed", a, n_samples, audio_stride, h_probs, max_probs, h_probs_out);
    });
}
int mww_predict_clip_remote_mixed(mww_t *h, const uint8_t *src_audio, int n_samples, long long audio_stride, float *d_probs, int max_probs,
                                  int *h_probs_out, int n_tiles, void *cu_stream) {
    return with_mixed(h, "mww_predict_clip_remote_mixed", src_audio, [&](auto a) {
        if (int rc = refuse_multi(h, "mww_predict_clip_remote_mixed", "mww_predict_clip_remote_multi_mixed")) return rc;
        return predict_clip_remote_impl(h, "mww_predict_clip_remote_mixed", a, n_samples, audio_stride, &d_probs, &max_probs, h_probs_out,
                                        n_tiles, cu_stream);
    });
}
int mww_predict_clip_remote_multi_mixed(mww_t *h, const uint8_t *src_audio, int n_samples, long long audio_stride, float *const *d_probs,
                                        const int *max_probs, int *h_probs_out, int n_tiles, void *cu_stream) {
    return with_mixed(h, "mww_predict_clip_remote_multi_mixed", src_audio, [&](auto a) {
        return predict_clip_remote_impl(h, "mww_predict_clip_remote_multi_mixed", a, n_samples, audio_stride, d_probs, max_probs,
                                        h_probs_out, n_tiles, cu_stream);
    });
}

// ---- host memory next to the GPU ---------------------------------------------------------------------------------
namespace {

int device_numa_node(int device) {
    char bdf[32] = {0};
    if (cudaDeviceGetPCIBusId(bdf, sizeof bdf, device) != cudaSuccess) { cudaGetLastError(); return -1; }
    for (char *c = bdf; *c; ++c) if (*c >= 'A' && *c <= 'F') *c = (char)(*c - 'A' + 'a');
    char path[128];
    snprintf(path, sizeof path, "/sys/bus/pci/devices/%s/numa_node", bdf);
    FILE *f = fopen(path, "r");
    if (!f) return -1;
    int node = -1;
    if (fscanf(f, "%d", &node) != 1) node = -1;
    fclose(f);
    return node;
}

// CPUs of a NUMA node that the calling thread is allowed to run on (empty set: unknown node / nothing allowed)
bool node_cpus(int node, cpu_set_t *out) {
    CPU_ZERO(out);
    if (node < 0) return false;
    char path[96];
    snprintf(path, sizeof path, "/sys/devices/system/node/node%d/cpulist", node);
    FILE *f = fopen(path, "r");
    if (!f) return false;
    char buf[4096];
    const bool got = fgets(buf, sizeof buf, f) != nullptr;
    fclose(f);
    if (!got) return false;
    cpu_set_t allowed;
    CPU_ZERO(&allowed);
    if (sched_getaffinity(0, sizeof allowed, &allowed) != 0) return false;
    int n = 0;
    for (char *p = buf; *p;) {
        char *end;
        const long a = strtol(p, &end, 10);
        if (end == p) break;
        long b = a;
        if (*end == '-') { p = end + 1; b = strtol(p, &end, 10); }
        for (long c = a; c <= b && c < CPU_SETSIZE; ++c)
            if (CPU_ISSET(c, &allowed)) { CPU_SET(c, out); ++n; }
        p = *end == ',' ? end + 1 : end;
        if (*end != ',') break;
    }
    return n > 0;
}

// MPOL_PREFERRED on one node for the calling thread (best effort: containers may forbid the syscall)
void prefer_node(int node) {
#ifdef SYS_set_mempolicy
    if (node < 0 || node >= 1024) { syscall(SYS_set_mempolicy, 0 /* MPOL_DEFAULT */, nullptr, 0); return; }
    unsigned long mask[16] = {0};
    mask[node / (8 * sizeof(unsigned long))] |= 1ul << (node % (8 * sizeof(unsigned long)));
    syscall(SYS_set_mempolicy, 1 /* MPOL_PREFERRED */, mask, sizeof mask * 8);
#else
    (void)node;
#endif
}

}  // namespace

int mww_bind_host_thread(int device, int *numa_node_out) {
    const int node = device_numa_node(device);
    if (numa_node_out) *numa_node_out = node;
    cpu_set_t cpus;
    if (!node_cpus(node, &cpus)) return MWW_OK;          // unknown topology: leave the thread where it is
    if (sched_setaffinity(0, sizeof cpus, &cpus) != 0) { g_create_error = "mww_bind_host_thread: sched_setaffinity failed"; return MWW_EINVAL; }
    return MWW_OK;
}

namespace {
int host_alloc_impl(size_t bytes, int device, unsigned flags, void **h_ptr, int *numa_node_out);
}
int mww_host_alloc(size_t bytes, int device, void **h_ptr, int *numa_node_out) {
    return host_alloc_impl(bytes, device, cudaHostAllocPortable, h_ptr, numa_node_out);
}
int mww_host_alloc_wc(size_t bytes, int device, void **h_ptr, int *numa_node_out) {
    return host_alloc_impl(bytes, device, cudaHostAllocPortable | cudaHostAllocWriteCombined, h_ptr, numa_node_out);
}
namespace {
int host_alloc_impl(size_t bytes, int device, unsigned flags, void **h_ptr, int *numa_node_out) {
    if (!h_ptr || bytes == 0) { g_create_error = "mww_host_alloc: bad argument"; return MWW_EINVAL; }
    *h_ptr = nullptr;
    DeviceGuard guard(device);
    if (guard.err != cudaSuccess) return ipc_fail("mww_host_alloc: cudaSetDevice", guard.err);
    const int node = device_numa_node(device);
    if (numa_node_out) *numa_node_out = node;
    // pages are placed where the pinning thread runs: move this thread next to the GPU for the duration of the allocation
    cpu_set_t before, cpus;
    CPU_ZERO(&before);
    const bool have_before = sched_getaffinity(0, sizeof before, &before) == 0;
    const bool moved = have_before && node_cpus(node, &cpus) && sched_setaffinity(0, sizeof cpus, &cpus) == 0;
    if (moved) prefer_node(node);
    void *p = nullptr;
    const cudaError_t e = cudaHostAlloc(&p, bytes, flags);
    if (moved) { prefer_node(-1); sched_setaffinity(0, sizeof before, &before); }
    if (e != cudaSuccess) return ipc_fail("mww_host_alloc: cudaHostAlloc", e);
    *h_ptr = p;
    return MWW_OK;
}
}  // namespace

int mww_host_free(void *h_ptr) {
    if (!h_ptr) return MWW_OK;
    const cudaError_t e = cudaFreeHost(h_ptr);
    return e == cudaSuccess ? MWW_OK : ipc_fail("mww_host_free", e);
}

namespace {
// one model's NN state to / from the host; the exported ring layout is always the canonical oldest-first one
int get_model_state(mww_t *h, Model &m, void *h_nn, void *h_pending) {
    const size_t M = (size_t)m.members();
    if (h_nn) {
        if (int rc = canonicalise_rings(h, m, nullptr)) return rc;
        CU(h, cudaDeviceSynchronize());
        if (M > 0) CU(h, cudaMemcpy(h_nn, m.d_nn_state, M * m.state_bytes(), cudaMemcpyDeviceToHost));
    }
    if (h_pending && M > 0) CU(h, cudaMemcpy(h_pending, m.d_pend, M * m.pend_bytes(), cudaMemcpyDeviceToHost));
    return MWW_OK;
}
int set_model_state(mww_t *h, Model &m, const void *h_nn, const void *h_pending, int pending_rows) {
    const size_t M = (size_t)m.members();
    note_state_set(h, m, h_nn, h_pending, pending_rows);
    if (h_nn) {
        if (M > 0) CU(h, cudaMemcpy(m.d_nn_state, h_nn, M * m.state_bytes(), cudaMemcpyHostToDevice));
        m.live_heads = LiveHeads{};
    }
    if (h_pending && M > 0) CU(h, cudaMemcpy(m.d_pend, h_pending, M * m.pend_bytes(), cudaMemcpyHostToDevice));
    m.n_pend = pending_rows;
    return MWW_OK;
}
}  // namespace

int mww_get_state(mww_t *h, int16_t *h_carry, uint32_t *h_estimate, void *h_nn, void *h_pending) {
    if (!h) return MWW_EINVAL;
    if (h_nn || h_pending)
        if (int rc = refuse_multi(h, "mww_get_state", "mww_get_model_state for the NN state")) return rc;
    ENTER_STATEFUL(h);
    CU(h, cudaDeviceSynchronize());
    const size_t S = (size_t)h->n_streams;
    if (h_carry) CU(h, cudaMemcpy(h_carry, h->d_carry, S * kWindow * 2, cudaMemcpyDeviceToHost));
    if (h_estimate) CU(h, cudaMemcpy(h_estimate, h->d_estimate, S * kNumChannels * 4, cudaMemcpyDeviceToHost));
    if (!h_nn && !h_pending) return MWW_OK;
    if (h->models.empty()) return fail(h, MWW_EINVAL, "frontend-only handle has no NN state");
    return get_model_state(h, h->models[0], h_nn, h_pending);
}

int mww_set_state(mww_t *h, const int16_t *h_carry, int frontend_buffered, const uint32_t *h_estimate, const void *h_nn,
                  const void *h_pending, int pending_rows) {
    if (!h) return MWW_EINVAL;
    if (h_nn || h_pending || pending_rows != 0)
        if (int rc = refuse_multi(h, "mww_set_state", "mww_set_model_state for the NN state and pending rows")) return rc;
    const int stride = h->models.empty() ? okay_nabu_arch().stride : h->models[0].G.stride;
    if (frontend_buffered < 0 || frontend_buffered >= kWindow || pending_rows < 0 || pending_rows > stride - 1)
        return fail(h, MWW_EINVAL, "mww_set_state: counters out of range");
    ENTER(h);
    CU(h, cudaDeviceSynchronize());
    const size_t S = (size_t)h->n_streams;
    if (h_carry) CU(h, cudaMemcpy(h->d_carry, h_carry, S * kWindow * 2, cudaMemcpyHostToDevice));
    if (h_estimate) CU(h, cudaMemcpy(h->d_estimate, h_estimate, S * kNumChannels * 4, cudaMemcpyHostToDevice));
    if ((h_nn || h_pending) && h->models.empty()) return fail(h, MWW_EINVAL, "frontend-only handle has no NN state");
    // several models: each keeps its own pending rows (mww_set_model_state)
    if (h->models.size() == 1)
        if (int rc = set_model_state(h, h->models[0], h_nn, h_pending, pending_rows)) return rc;
    h->used = frontend_buffered;
    return MWW_OK;
}

int mww_get_model_state(mww_t *h, int k, void *h_nn, void *h_pending) {
    if (!h) return MWW_EINVAL;
    if (k < 0 || k >= (int)h->models.size()) return fail(h, MWW_EINVAL, "mww_get_model_state: model index out of range");
    ENTER_STATEFUL(h);
    CU(h, cudaDeviceSynchronize());
    return get_model_state(h, h->models[k], h_nn, h_pending);
}

int mww_set_model_state(mww_t *h, int k, const void *h_nn, const void *h_pending, int pending_rows) {
    if (!h) return MWW_EINVAL;
    if (k < 0 || k >= (int)h->models.size()) return fail(h, MWW_EINVAL, "mww_set_model_state: model index out of range");
    Model &m = h->models[k];
    if (pending_rows < 0 || pending_rows > m.G.stride - 1) return fail(h, MWW_EINVAL, "mww_set_model_state: pending_rows out of range");
    ENTER(h);
    CU(h, cudaDeviceSynchronize());
    return set_model_state(h, m, h_nn, h_pending, pending_rows);
}

int mww_set_model_streams(mww_t *h, int k, const int32_t *h_ids, int n, void *cu_stream) {
    if (!h) return MWW_EINVAL;
    if (k < 0 || k >= (int)h->models.size()) return fail(h, MWW_EINVAL, "mww_set_model_streams: model index out of range");
    if (h_ids && (n < 0 || n > h->n_streams || !valid_stream_set(h_ids, n, h->n_streams)))
        return fail(h, MWW_EINVAL, "mww_set_model_streams: stream ids must be strictly increasing and in [0, n_streams)");
    ENTER_STATEFUL(h);
    cudaStream_t st = static_cast<cudaStream_t>(cu_stream);
    Model &m = h->models[k];
    MemberState ns;
    if (int rc = alloc_members(h, m, h_ids, n, &ns)) return rc;
    // new member j takes the rows of old compact index old_index[j]; the joiners (-1) get fresh state.  Every model's ring
    // rotation is the same for all its streams, so rows copied as they are stay valid while the rings are rotated.
    const int M = (int)ns.mem.ids.size();
    std::vector<int32_t> old_index(M), joiners;
    for (int j = 0; j < M; ++j) {
        const int s = ns.mem.ids[j];
        const int o = lower_bound_ids(m.mem.ids.data(), m.members(), s);
        old_index[j] = o < m.members() && m.mem.ids[o] == s ? o : -1;
        if (old_index[j] < 0) joiners.push_back(j);
    }
    std::vector<int32_t> maps(old_index);
    maps.insert(maps.end(), joiners.begin(), joiners.end());
    int32_t *d_maps = nullptr;
    cudaError_t e = maps.empty() ? cudaSuccess : cudaMalloc(&d_maps, maps.size() * sizeof(int32_t));
    if (e == cudaSuccess && d_maps) e = cudaMemcpyAsync(d_maps, maps.data(), maps.size() * sizeof(int32_t), cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess && (int)joiners.size() < M) {
        e = launch_remap_rows(ns.d_nn_state, m.d_nn_state, m.state_bytes(), d_maps, M, h->sm_count, st);
        if (e == cudaSuccess) e = launch_remap_rows(ns.d_pend, m.d_pend, m.pend_bytes(), d_maps, M, h->sm_count, st);
        if (e == cudaSuccess) h->launches += 2;
    }
    int rc = e == cudaSuccess ? MWW_OK : cuda_fail(h, e, "mww_set_model_streams: state remap");
    if (rc == MWW_OK && !joiners.empty()) rc = reset_nn_by_id(h, m, ns.d_nn_state, ns.d_pend, d_maps + M, (int)joiners.size(), M, st);
    // the old buffers (and the id maps) are freed only once the remap that reads them is done
    if (cudaError_t s = cudaStreamSynchronize(st)) if (rc == MWW_OK) rc = cuda_fail(h, s, "cudaStreamSynchronize");
    cudaFree(d_maps);
    if (rc != MWW_OK) { ns.release(); return rc; }
    cudaFree(m.mem.d_ids); cudaFree(m.mem.d_inv); cudaFree(m.d_nn_state); cudaFree(m.d_pend);
    m.mem = std::move(ns.mem);
    m.d_nn_state = ns.d_nn_state;
    m.d_pend = ns.d_pend;
    return MWW_OK;
}

int mww_get_model_streams(const mww_t *h, int k, int32_t *h_ids, int max_ids, int *n_out) {
    if (!h || k < 0 || k >= (int)h->models.size() || max_ids < 0 || (max_ids > 0 && !h_ids)) return MWW_EINVAL;
    const std::vector<int32_t> &ids = h->models[k].mem.ids;
    std::copy(ids.begin(), ids.begin() + std::min<size_t>(ids.size(), (size_t)max_ids), h_ids);
    if (n_out) *n_out = (int)ids.size();
    return MWW_OK;
}

int mww_copy_nn_state(mww_t *dst, const int32_t *h_dst_ids, const mww_t *src_c, const int32_t *h_src_ids, int n, void *cu_stream) {
    if (!dst) return MWW_EINVAL;
    if (int rc = refuse_multi(dst, "mww_copy_nn_state", "a one-model handle")) return rc;
    if (src_c && src_c->models.size() > 1) return fail(dst, MWW_EINVAL, "mww_copy_nn_state: the source handle carries several models");
    if (src_c && !all_streams(src_c)) return fail(dst, MWW_EINVAL, "mww_copy_nn_state: the source model runs on a subset of the streams");
    // canonicalising the source's rings changes their layout, not the state they hold
    mww_t *src = const_cast<mww_t *>(src_c);
    if (!src || n < 0 || (n > 0 && (!h_dst_ids || !h_src_ids))) return fail(dst, MWW_EINVAL, "mww_copy_nn_state: bad arguments");
    if (src->device != dst->device) return fail(dst, MWW_EINVAL, "mww_copy_nn_state: the handles are on different devices");
    if (src->models.empty() || dst->models.empty()) return fail(dst, MWW_EINVAL, "mww_copy_nn_state: frontend-only handle has no NN state");
    Model &ms = src->models[0], &md = dst->models[0];
    if (ms.model_hash != md.model_hash || ms.quantized() != md.quantized() || ms.G.state_elems != md.G.state_elems)
        return fail(dst, MWW_EINVAL, "mww_copy_nn_state: the handles were created from different models");
    if (ms.n_pend != 0 || md.n_pend != 0) return fail(dst, MWW_EINVAL, "mww_copy_nn_state: a handle holds pending rows");
    for (int i = 0; i < n; ++i)
        if (h_dst_ids[i] < 0 || h_dst_ids[i] >= dst->n_streams || h_src_ids[i] < 0 || h_src_ids[i] >= src->n_streams)
            return fail(dst, MWW_EINVAL, "mww_copy_nn_state: stream id out of range");
    ENTER_STATEFUL(dst);
    if (src->poisoned) return fail(dst, MWW_ECUDA, "mww_copy_nn_state: the source handle needs mww_reset(h, NULL, 0, stream)");
    cudaStream_t st = static_cast<cudaStream_t>(cu_stream);
    int rc = canonicalise_rings(src, ms, st);
    if (rc) return fail(dst, rc, "mww_copy_nn_state: " + src->err);
    if (dst != src && (rc = canonicalise_rings(dst, md, st)) != MWW_OK) return rc;
    md.tc_rows_bounded = md.tc_rows_bounded && ms.tc_rows_bounded;
    const size_t bytes = (size_t)md.G.state_elems * md.elem_size();
    char *d = static_cast<char *>(md.d_nn_state);
    const char *s = static_cast<const char *>(ms.d_nn_state);
    for (int i = 0; i < n; ++i) {
        if (dst == src && h_dst_ids[i] == h_src_ids[i]) continue;     // same bytes: nothing to copy (and memcpy needs disjoint ranges)
        CU(dst, cudaMemcpyAsync(d + (size_t)h_dst_ids[i] * bytes, s + (size_t)h_src_ids[i] * bytes, bytes, cudaMemcpyDeviceToDevice, st));
    }
    return MWW_OK;
}

// ---- stream records: a stream's whole state between handles (layout and index math: mww_records.h) ------------------
namespace {
static_assert(kMaxModels == kRecordMaxModels, "one bit of the member mask per model");

RecordModel record_model(const Model &m) { return RecordModel{(long long)m.state_bytes(), (long long)m.pend_bytes()}; }

RecordLayout handle_record_layout(const mww_t *h) {
    RecordModel rm[kMaxModels];
    for (size_t k = 0; k < h->models.size(); ++k) rm[k] = record_model(h->models[k]);
    return record_layout(rm, (int)h->models.size());
}

void fill_stream_layout(const mww_t *h, mww_stream_layout *o) {
    memset(o, 0, sizeof *o);
    o->record_bytes = handle_record_layout(h).record_bytes;
    o->n_models = (int)h->models.size();
    o->frontend_buffered = h->used;
    o->hop_samples = h->hop;
    for (size_t k = 0; k < h->models.size(); ++k) {
        const Model &m = h->models[k];
        o->pending_rows[k] = m.n_pend;
        o->model_hash[k] = record_model_hash(m.model_hash, m.quantized(), m.G.state_elems);
        o->rows_are_features[k] = m.tc_rows_bounded;
    }
}

// model k's ring state and pending rows, with the rotation live calls have left its rings in.  Only the compiled-in
// okay_nabu kernels rotate (blocks 0..3 and the head ring, after the first-conv ring); every other kind keeps canonical
// rings, so its state is one plain span.
RecordJob model_record_job(const RecordLayout &L, int k, const Model &m) {
    RecordJob J = record_job_model(L, k, record_model(m));
    J.zero_fresh = !m.quantized();
    if (m.compiled()) {
        const int es = (int)m.elem_size();
        int off = 2 * kNumChannels;
        for (int i = 0; i < 5; ++i) {
            record_add_ring(&J, off * es, live_ring_cols(i) * es, kLiveRingRows[i], m.live_heads.h[i]);
            off += kLiveRingRows[i] * live_ring_cols(i);
        }
    }
    return J;
}

// argument checks shared by export and import; returns MWW_OK or the failure already recorded on h
int check_record_args(mww_t *h, const char *who, const int32_t *h_ids, int n, const void *d_records) {
    if (n < 0 || (n > 0 && (!h_ids || !d_records))) return fail(h, MWW_EINVAL, std::string(who) + ": bad arguments");
    if (reinterpret_cast<uintptr_t>(d_records) % 16 != 0) return fail(h, MWW_EINVAL, std::string(who) + ": the records must be 16-byte aligned");
    for (int i = 0; i < n; ++i)
        if (h_ids[i] < 0 || h_ids[i] >= h->n_streams) return fail(h, MWW_EINVAL, std::string(who) + ": stream id out of range");
    return MWW_OK;
}
}  // namespace

int mww_stream_layout_get(const mww_t *h, mww_stream_layout *out) {
    if (!h || !out) return MWW_EINVAL;
    fill_stream_layout(h, out);
    return MWW_OK;
}

namespace {
// the device work of mww_export_streams, into records `pitch` bytes apart (h->d_ids holds the n ids)
int pack_stream_records(mww_t *h, int n, void *d_records, long long pitch, cudaStream_t st) {
    const RecordLayout L = handle_record_layout(h);
    const void *fe[kRecordMaxParts] = {nullptr, h->d_carry, h->d_estimate};
    CU(h, launch_pack_streams(record_job_frontend(L), d_records, pitch, h->d_ids, n, fe, nullptr, h->sm_count, st));
    h->launches += 1;
    for (size_t k = 0; k < h->models.size(); ++k) {
        const Model &m = h->models[k];
        const void *nn[kRecordMaxParts] = {m.d_nn_state, m.d_pend, nullptr};
        CU(h, launch_pack_streams(model_record_job(L, (int)k, m), d_records, pitch, h->d_ids, n, nn, m.mem.d_inv, h->sm_count, st));
        h->launches += 1;
    }
    return MWW_OK;
}

// the host checks of mww_import_streams after the arguments: no id twice, and the records' layout fits the handle
int check_import_layout(mww_t *h, const char *who, const int32_t *h_ids, int n, const mww_stream_layout *layout) {
    std::vector<uint8_t> listed((size_t)h->n_streams, 0);
    for (int i = 0; i < n; ++i) {
        if (listed[(size_t)h_ids[i]]) return fail(h, MWW_EINVAL, std::string(who) + ": a stream id is listed twice");
        listed[(size_t)h_ids[i]] = 1;
    }
    mww_stream_layout mine;
    fill_stream_layout(h, &mine);
    int which = -1;
    if (const char *field = stream_layout_mismatch(*layout, mine, &which))
        return fail(h, MWW_EINVAL, std::string(who) + ": the records' " + field +
                                       (which >= 0 ? " of model " + std::to_string(which) : std::string()) + " differs from the handle's");
    return MWW_OK;
}

// the device work of mww_import_streams, from records `pitch` bytes apart; uploads the n ids to h->d_ids
int unpack_stream_records(mww_t *h, const int32_t *h_ids, int n, const void *d_records, long long pitch, const mww_stream_layout *layout,
                          cudaStream_t st) {
    if (int rc = ensure_ids(h, &h->d_cids, &h->cids_cap, n, st)) return rc;
    if (int rc = upload_ids(h, h_ids, n, st)) return rc;
    const RecordLayout L = handle_record_layout(h);
    void *fe[kRecordMaxParts] = {nullptr, h->d_carry, h->d_estimate};
    CU(h, launch_unpack_streams(record_job_frontend(L), d_records, pitch, h->d_ids, n, fe, nullptr, nullptr, h->sm_count, st));
    h->launches += 1;
    // records carry no audio history: the streams written start theirs afresh
    if (h->d_hist)
        if (int rc = fill_by_id(h, h->d_hist, (size_t)h->hist_cap * sizeof(int16_t), h->d_ids, n, h->n_streams, st)) return rc;
    for (size_t k = 0; k < h->models.size(); ++k) {
        Model &m = h->models[k];
        if (m.members() == 0) continue;
        void *nn[kRecordMaxParts] = {m.d_nn_state, m.d_pend, nullptr};
        // members the records hold no state for start fresh, as the joiners of mww_set_model_streams do: zeros (fp32, hybrid)
        // are written by the unpack kernel, zero points (int8) by the model's fill kernel over the list it leaves in d_cids
        const RecordJob J = model_record_job(L, (int)k, m);
        CU(h, launch_unpack_streams(J, d_records, pitch, h->d_ids, n, nn, m.mem.d_inv, J.zero_fresh ? nullptr : h->d_cids, h->sm_count, st));
        h->launches += 1;
        if (!J.zero_fresh)
            if (int rc = reset_nn_by_id(h, m, m.d_nn_state, m.d_pend, h->d_cids, n, m.members(), st)) return rc;
        m.tc_rows_bounded = m.tc_rows_bounded && layout->rows_are_features[k];
    }
    return MWW_OK;
}
}  // namespace

int mww_export_streams(mww_t *h, const int32_t *h_ids, int n, void *d_records, mww_stream_layout *out, void *cu_stream) {
    if (!h) return MWW_EINVAL;
    if (resampling(h)) return fail(h, MWW_EUNSUPPORTED, "mww_export_streams: stream records do not carry resampler history (input rate != 16000, or per-stream rates)");
    if (int rc = check_record_args(h, "mww_export_streams", h_ids, n, d_records)) return rc;
    ENTER_STATEFUL(h);
    if (out) fill_stream_layout(h, out);
    if (n == 0) return MWW_OK;
    cudaStream_t st = static_cast<cudaStream_t>(cu_stream);
    if (int rc = upload_ids(h, h_ids, n, st)) return rc;
    return pack_stream_records(h, n, d_records, handle_record_layout(h).record_bytes, st);
}

int mww_import_streams(mww_t *h, const int32_t *h_ids, int n, const void *d_records, const mww_stream_layout *layout, void *cu_stream) {
    if (!h) return MWW_EINVAL;
    if (resampling(h)) return fail(h, MWW_EUNSUPPORTED, "mww_import_streams: stream records do not carry resampler history (input rate != 16000, or per-stream rates)");
    if (!layout) return fail(h, MWW_EINVAL, "mww_import_streams: bad arguments");
    if (int rc = check_record_args(h, "mww_import_streams", h_ids, n, d_records)) return rc;
    if (int rc = check_import_layout(h, "mww_import_streams", h_ids, n, layout)) return rc;
    ENTER_STATEFUL(h);
    if (n == 0) return MWW_OK;
    cudaStream_t st = static_cast<cudaStream_t>(cu_stream);
    return unpack_stream_records(h, h_ids, n, d_records, handle_record_layout(h).record_bytes, layout, st);
}

// ---- resampled stream records: stream records plus the resampler history (rule: include/mww.h) -------------------------
namespace {
void fill_resampler_layout(const mww_t *h, mww_resampler_layout *o) {
    memset(o, 0, sizeof *o);
    o->resampler_off = handle_record_layout(h).record_bytes;
    o->record_bytes = o->resampler_off + kRecordResamplerPart;
    o->rate = h->per_rate ? MWW_RATE_PER_STREAM : h->rs.rate;
    o->inputs_seen = h->rs_seen;
    o->samples16_seen = h->per_rate ? h->rs_seen : resample_outputs(h->rs_seen, h->rs.L, h->rs.M);
}

int stream_rate_of(const mww_t *h, int id) { return h->per_rate ? h->stream_rate[(size_t)id] : h->rs.rate; }

// N mod M of a stream at plan P on the counters of a resampler layout: N = inputs_seen on a single-rate handle,
// floor(t M / L) with per-stream rates
long long rate_phase(const mww_resampler_layout &r, const ResamplePlan &P) {
    const long long N = r.rate == MWW_RATE_PER_STREAM ? resample_inputs(r.samples16_seen, P.L, P.M) : r.inputs_seen;
    return N % P.M;
}
}  // namespace

int mww_get_resampler_layout(const mww_t *h, mww_resampler_layout *out) {
    if (!h || !out) return MWW_EINVAL;
    fill_resampler_layout(h, out);
    return MWW_OK;
}

int mww_export_resampled_streams(mww_t *h, const int32_t *h_ids, int n, void *d_records, mww_stream_layout *out,
                                 mww_resampler_layout *rs_out, int32_t *h_rates_out, void *cu_stream) {
    if (!h) return MWW_EINVAL;
    if (int rc = check_record_args(h, "mww_export_resampled_streams", h_ids, n, d_records)) return rc;
    ENTER_STATEFUL(h);
    if (out) fill_stream_layout(h, out);
    mww_resampler_layout R;
    fill_resampler_layout(h, &R);
    if (rs_out) *rs_out = R;
    if (h_rates_out)
        for (int i = 0; i < n; ++i) h_rates_out[i] = stream_rate_of(h, h_ids[i]);
    if (n == 0) return MWW_OK;
    cudaStream_t st = static_cast<cudaStream_t>(cu_stream);
    if (int rc = upload_ids(h, h_ids, n, st)) return rc;
    if (int rc = pack_stream_records(h, n, d_records, R.record_bytes, st)) return rc;
    const void *rs[kRecordMaxParts] = {h->d_rs_hist, nullptr, nullptr};
    CU(h, launch_pack_streams(record_job_resampler(R.resampler_off, h->rs_hist_stride), d_records, R.record_bytes, h->d_ids, n, rs, nullptr,
                              h->sm_count, st));
    h->launches += 1;
    return MWW_OK;
}

int mww_import_resampled_streams(mww_t *h, const int32_t *h_ids, int n, const void *d_records, const mww_stream_layout *layout,
                                 const mww_resampler_layout *rs_layout, const int32_t *h_rates, void *cu_stream) {
    static const char *who = "mww_import_resampled_streams";
    if (!h) return MWW_EINVAL;
    if (!layout || !rs_layout || (n > 0 && !h_rates)) return fail(h, MWW_EINVAL, std::string(who) + ": bad arguments");
    if (int rc = check_record_args(h, who, h_ids, n, d_records)) return rc;
    if (int rc = check_import_layout(h, who, h_ids, n, layout)) return rc;
    mww_resampler_layout mine;
    fill_resampler_layout(h, &mine);
    const mww_resampler_layout &src = *rs_layout;
    const auto refuse = [&](const std::string &why) { return fail(h, MWW_EINVAL, std::string(who) + ": " + why); };
    if (src.record_bytes != mine.record_bytes) return refuse("the records' record_bytes differs from the handle's");
    if (src.resampler_off != mine.resampler_off) return refuse("the records' resampler_off differs from the handle's");
    ResamplePlan Psrc;
    if (src.rate != MWW_RATE_PER_STREAM && !resample_plan(src.rate, &Psrc)) return refuse("the records' rate is not an input rate");
    if (src.inputs_seen < 0 || src.samples16_seen < 0 || src.samples16_seen > (1ll << 50))
        return refuse("the records' counters are out of range");
    // each rate's phase in the records and in the handle, once per rate; the message is built only for a refusal
    long long phase[kNumRates][2];
    ResamplePlan plan[kNumRates];
    for (int i = 0; i < kNumRates; ++i) {
        resample_plan(kResampleRates[i], &plan[i]);
        phase[i][0] = rate_phase(src, plan[i]);
        phase[i][1] = rate_phase(mine, plan[i]);
    }
    for (int i = 0; i < n; ++i) {
        const int id = h_ids[i], r = h_rates[i], dst_rate = stream_rate_of(h, id), slot = rate_slot(r);
        if ((src.rate == MWW_RATE_PER_STREAM || r == src.rate) && r == dst_rate && phase[slot][0] == phase[slot][1]) continue;
        const std::string stream = "stream " + std::to_string(id) + " (h_rates[" + std::to_string(i) + "] = " + std::to_string(r) + ")";
        if (src.rate != MWW_RATE_PER_STREAM && r != src.rate)
            return refuse(stream + ": the rate is not the records' rate " + std::to_string(src.rate));
        if (r != dst_rate) return refuse(stream + ": the rate is not the handle's rate " + std::to_string(dst_rate) + " for it");
        return refuse(stream + ": phase mismatch at " + std::to_string(r) + " Hz: the records' N mod " + std::to_string(plan[slot].M) + " = " +
                      std::to_string(phase[slot][0]) + ", the handle's " + std::to_string(phase[slot][1]));
    }
    ENTER_STATEFUL(h);
    if (n == 0) return MWW_OK;
    cudaStream_t st = static_cast<cudaStream_t>(cu_stream);
    if (int rc = unpack_stream_records(h, h_ids, n, d_records, mine.record_bytes, layout, st)) return rc;
    void *rs[kRecordMaxParts] = {h->d_rs_hist, nullptr, nullptr};
    CU(h, launch_unpack_streams(record_job_resampler(mine.resampler_off, h->rs_hist_stride), d_records, mine.record_bytes, h->d_ids, n, rs,
                                nullptr, nullptr, h->sm_count, st));
    h->launches += 1;
    return MWW_OK;
}

// ---- audio history: the last C 16 kHz samples of every stream (rule: include/mww.h; ring and kernels: mww_history.{h,cu}) ----
int mww_set_audio_history(mww_t *h, int capacity, void *cu_stream) {
    if (!h) return MWW_EINVAL;
    if (!history_capacity_ok(capacity))
        return fail(h, MWW_EINVAL, "mww_set_audio_history: the capacity must be 0 or a multiple of 8 in [8, " + std::to_string(kHistoryMaxCapacity) + "]");
    ENTER_STATEFUL(h);
    cudaStream_t st = static_cast<cudaStream_t>(cu_stream);
    int16_t *ring = nullptr;
    if (capacity > 0) {
        const size_t bytes = (size_t)h->n_streams * capacity * sizeof(int16_t);
        cudaError_t e = cudaMalloc(&ring, bytes);
        if (e != cudaSuccess) {
            cudaGetLastError();
            return fail(h, e == cudaErrorMemoryAllocation ? MWW_ENOMEM : MWW_ECUDA, std::string("mww_set_audio_history: ") + cudaGetErrorString(e));
        }
        if ((e = cudaMemsetAsync(ring, 0, bytes, st)) != cudaSuccess) { cudaFree(ring); return cuda_fail(h, e, "mww_set_audio_history"); }
    }
    // earlier calls on the stream may still append to the old ring
    if (h->d_hist) {
        if (cudaError_t e = cudaStreamSynchronize(st)) { cudaFree(ring); return cuda_fail(h, e, "cudaStreamSynchronize"); }
        cudaFree(h->d_hist);
    }
    h->d_hist = ring;
    h->hist_cap = capacity;
    h->hist_seen = 0;
    return MWW_OK;
}

}  // extern "C"

namespace mww {
HistoryRing history_ring(const mww_t *h) { return HistoryRing{h->d_hist, h->hist_cap, h->hist_seen, h->n_streams, h->sm_count, h->poisoned}; }
}  // namespace mww

extern "C" {

int mww_get_audio_history(const mww_t *h, int *capacity, long long *samples_seen) {
    if (!h) return MWW_EINVAL;
    if (capacity) *capacity = h->hist_cap;
    if (samples_seen) *samples_seen = h->hist_seen;
    return MWW_OK;
}

namespace {
// the checks both reads share, before any device work; ids are the caller's (host or device) list
int check_history_read(mww_t *h, const char *who, const void *ids, int n, int n_samples, const int16_t *d_out, long long out_stride) {
    if (!h->d_hist) return fail(h, MWW_EINVAL, std::string(who) + ": the handle keeps no audio history (mww_set_audio_history)");
    if (n < 0 || n_samples < 0 || n_samples > h->hist_cap || out_stride < n_samples)
        return fail(h, MWW_EINVAL, std::string(who) + ": needs n >= 0, 0 <= n_samples <= capacity and out_stride >= n_samples");
    if (n > 0 && n_samples > 0 && (!ids || !d_out)) return fail(h, MWW_EINVAL, std::string(who) + ": NULL ids or output");
    return MWW_OK;
}
int read_history(mww_t *h, const int32_t *d_ids, int n, int n_samples, int16_t *d_out, long long out_stride, cudaStream_t st) {
    CU(h, launch_history_read(h->d_hist, h->hist_cap, h->hist_seen, d_ids, n, h->n_streams, n_samples, d_out, out_stride, h->sm_count, st));
    h->launches += 1;
    return MWW_OK;
}
}  // namespace

int mww_read_audio_history(mww_t *h, const int32_t *h_ids, int n, int n_samples, int16_t *d_out, long long out_stride, void *cu_stream) {
    if (!h) return MWW_EINVAL;
    if (int rc = check_history_read(h, "mww_read_audio_history", h_ids, n, n_samples, d_out, out_stride)) return rc;
    for (int i = 0; n_samples > 0 && i < n; ++i)
        if (h_ids[i] < 0 || h_ids[i] >= h->n_streams) return fail(h, MWW_EINVAL, "mww_read_audio_history: stream id out of range");
    ENTER_STATEFUL(h);
    if (n == 0 || n_samples == 0) return MWW_OK;
    cudaStream_t st = static_cast<cudaStream_t>(cu_stream);
    if (int rc = upload_ids(h, h_ids, n, st)) return rc;
    return read_history(h, h->d_ids, n, n_samples, d_out, out_stride, st);
}

int mww_read_audio_history_device_ids(mww_t *h, const int32_t *d_ids, int n, int n_samples, int16_t *d_out, long long out_stride, void *cu_stream) {
    if (!h) return MWW_EINVAL;
    if (int rc = check_history_read(h, "mww_read_audio_history_device_ids", d_ids, n, n_samples, d_out, out_stride)) return rc;
    ENTER_STATEFUL(h);
    if (n == 0 || n_samples == 0) return MWW_OK;
    return read_history(h, d_ids, n, n_samples, d_out, out_stride, static_cast<cudaStream_t>(cu_stream));
}

int mww_read_audio_history_at(mww_t *h, const int32_t *d_ids, const long long *d_ends, int n, int n_samples, int16_t *d_out, long long out_stride,
                              void *cu_stream) {
    if (!h) return MWW_EINVAL;
    const char *who = "mww_read_audio_history_at";
    if (int rc = check_history_read(h, who, d_ids, n, n_samples, d_out, out_stride)) return rc;
    if (n > 0 && n_samples > 0 && !d_ends) return fail(h, MWW_EINVAL, std::string(who) + ": NULL ends");
    ENTER_STATEFUL(h);
    if (n == 0 || n_samples == 0) return MWW_OK;
    CU(h, launch_history_read_at(h->d_hist, h->hist_cap, h->hist_seen, d_ids, d_ends, n, h->n_streams, n_samples, d_out, out_stride, h->sm_count,
                                 static_cast<cudaStream_t>(cu_stream)));
    h->launches += 1;
    return MWW_OK;
}

int mww_write_audio_history(mww_t *h, const int32_t *h_ids, int n, int n_samples, const int16_t *d_in, long long in_stride, void *cu_stream) {
    if (!h) return MWW_EINVAL;
    const char *who = "mww_write_audio_history";
    if (!h->d_hist) return fail(h, MWW_EINVAL, std::string(who) + ": the handle keeps no audio history (mww_set_audio_history)");
    if (n < 0 || n_samples < 0 || n_samples > kHistoryMaxCapacity || in_stride < n_samples)
        return fail(h, MWW_EINVAL, std::string(who) + ": needs n >= 0, 0 <= n_samples <= 2^22 and in_stride >= n_samples");
    if (n > 0 && (!h_ids || (n_samples > 0 && !d_in))) return fail(h, MWW_EINVAL, std::string(who) + ": NULL ids or input");
    std::vector<uint8_t> listed((size_t)h->n_streams, 0);
    for (int i = 0; i < n; ++i) {
        if (h_ids[i] < 0 || h_ids[i] >= h->n_streams) return fail(h, MWW_EINVAL, std::string(who) + ": stream id out of range");
        if (listed[(size_t)h_ids[i]]) return fail(h, MWW_EINVAL, std::string(who) + ": a stream id is listed twice");
        listed[(size_t)h_ids[i]] = 1;
    }
    ENTER_STATEFUL(h);
    if (n == 0) return MWW_OK;
    cudaStream_t st = static_cast<cudaStream_t>(cu_stream);
    if (int rc = upload_ids(h, h_ids, n, st)) return rc;
    CU(h, launch_history_write(h->d_hist, h->hist_cap, h->hist_seen, h->d_ids, n, n_samples, d_in, in_stride, h->sm_count, st));
    h->launches += 1;
    return MWW_OK;
}

}  // extern "C"
