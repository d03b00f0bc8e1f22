// mww_capi.cu -- the extern "C" boundary declared in include/mww.h.
//
// Host-side orchestration only: model-container parsing, weight/table upload, per-stream state,
// stream tiling against a scratch budget, and the pipelined host-buffer path.  All arithmetic is
// in the kernels (mww_frontend.cu, mww_nn.cu, mww_nn_int8.cu); there is no CPU fallback.
#include <cuda_runtime.h>
#include <sched.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/syscall.h>
#include <unistd.h>

#include <algorithm>
#include <string>
#include <vector>

#include "../../include/mww.h"
#include "mww_kernels.h"
#include "mww_nn_i8_prep.h"
#include "mww_nn_tc.h"

using namespace mww;

namespace {

thread_local std::string g_create_error;

struct DirEntry { char name[48]; uint32_t dtype, ndim, shape[4]; uint64_t offset, nbytes; };
static_assert(sizeof(DirEntry) == 88, "container directory entry layout");

struct Tensor { const uint8_t *data = nullptr; uint32_t dtype = 0, ndim = 0, shape[4] = {0, 0, 0, 0}; uint64_t nbytes = 0; };

bool find_tensor(const uint8_t *blob, size_t n, const char *name, Tensor *out) {
    if (n < 24 || memcmp(blob, "MWWB200", 8) != 0) return false;
    uint32_t hdr[4];
    memcpy(hdr, blob + 8, 16);
    if (hdr[0] != 1) return false;
    const uint32_t count = hdr[1], dir_off = hdr[2];
    for (uint32_t i = 0; i < count; ++i) {
        if ((size_t)dir_off + (size_t)(i + 1) * sizeof(DirEntry) > n) return false;
        DirEntry e;
        memcpy(&e, blob + dir_off + (size_t)i * sizeof e, sizeof e);
        if (strncmp(e.name, name, 48) == 0) {
            if (e.offset > n || e.nbytes > n - e.offset) return false;
            out->data = blob + e.offset; out->dtype = e.dtype; out->ndim = e.ndim; out->nbytes = e.nbytes;
            memcpy(out->shape, e.shape, sizeof e.shape);
            return true;
        }
    }
    return false;
}

const int32_t kOkayNabuArch[30] = {32, 5, 3, 40, 4, 17, 64, 1, 5, 0, 0, 0, 64, 2, 7, 11, 0, 0, 64, 2, 9, 15, 0, 0, 64, 1, 23, 0, 0, 0};

}  // namespace

struct mww_handle {
    int device = 0, n_streams = 0, sm_count = 132;
    bool quantized = false;
    bool has_nn = true;
    uint64_t model_hash = 0;        // FNV-1a of the model container: mww_copy_nn_state only moves state between equal models
    std::string err;
    // constant tables
    uint8_t *d_tables = nullptr;
    FrontendParams P;
    // weights
    uint8_t *d_weights = nullptr;
    NnWeightsF32 W;
    TcWeights TW{};                 // fp32 okay_nabu: pre-split weights for the wgmma clip kernel (mww_nn_tc.cu)
    bool no_tc = false;             // MWW_NO_TC: keep the mma.sync clip kernel (A/B measurements)
    int live_variant = 3;           // MWW_LIVE_VARIANT: 3 = bulk-copy stages (default), 2 = warp-specialised with register loads, 1 = r01 kernel
    NnWeightsI8 Wq;
    float in_scale = 0.f, out_scale = 0.f;
    int in_zp = 0, out_zp = 0;
    // per-stream state
    int16_t *d_carry = nullptr;
    uint32_t *d_estimate = nullptr;
    void *d_nn_state = nullptr;     // float or int8 [S][state_elems]   (4176 for okay_nabu)
    void *d_pend = nullptr;         // float or int8 [S][pend_cap][40]  (2 rows for stride 3)
    int used = 0, n_pend = 0;
    int hop = kHop;                 // samples between feature windows (mww_set_window_step; 160 = the 10 ms of every shipped model)
    // geometry: the compiled-in okay_nabu kernels, or the run-time-geometry path (mww_nn_generic.cuh) for any other arch
    bool generic = false;
    GenArch G{};
    GenWeightsF32 GW{};
    GenWeightsI8 GQ{};
    int stride = 3;                 // feature rows per model step
    int pend_cap = 2;               // rows of the pending buffer
    int state_elems = kStateFloats; // ring-state elements per stream
    long long macs_per_step = 24800;
    // scratch
    uint32_t *d_v = nullptr; size_t v_bytes = 0;
    uint16_t *d_feat = nullptr; size_t feat_bytes = 0;
    size_t scratch_budget = (size_t)2048 << 20;
    int min_tile_streams = 2048;       // staged path: a tile never gets fewer streams than this (MWW_MIN_TILE_STREAMS)
    // host-buffer pipeline
    cudaStream_t st_h2d = nullptr, st_compute = nullptr, st_d2h = nullptr;
    cudaEvent_t ev_h2d[2] = {nullptr, nullptr}, ev_compute[2] = {nullptr, nullptr}, ev_d2h[2] = {nullptr, nullptr};
    cudaEvent_t ev_entry = nullptr, ev_exit = nullptr;
    bool staged_used = false;      // ev_compute[] have been recorded by an earlier staged call
    bool poisoned = false;
    int32_t *d_ids = nullptr; size_t ids_cap = 0;      // device copy of a host id list (mww_reset)         // a staged call failed half-way: per-stream state is inconsistent until mww_reset(all)
    int16_t *d_audio_tile[2] = {nullptr, nullptr}; size_t audio_tile_bytes = 0;
    float *d_probs_tile[2] = {nullptr, nullptr}; size_t probs_tile_bytes = 0;
    // live-step path: rings stay rotated between live calls (mww_nn_live.cuh); all streams advance in lockstep
    LiveHeads live_heads{};
    bool no_live = false, no_fuse = false;
    long long launches = 0;
    // optional per-kernel timing (mww_profile_*)
    bool profiling = false;
    std::vector<cudaEvent_t> prof_ev[4];   // start/stop pairs per kernel class
    std::vector<cudaEvent_t> tl_ev;        // last staged call while profiling: 4 events per tile (mww_timeline_read)
};

namespace {

int fail(mww_t *h, int code, const std::string &msg) {
    if (h) h->err = msg; else g_create_error = msg;
    return code;
}
int cuda_fail(mww_t *h, cudaError_t e, const char *what) {
    return fail(h, MWW_ECUDA, std::string(what) + ": " + cudaGetErrorString(e));
}
#define CU(h, call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return cuda_fail(h, e_, #call); } while (0)

size_t elem_size(const mww_t *h) { return h->quantized ? 1 : 4; }

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

int ensure_scratch(mww_t *h, size_t v_bytes, size_t feat_bytes) {
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

// streams per tile so that the K1->K2 scratch (when the call needs one) and the optional feature scratch fit the budget
int tile_streams(const mww_t *h, int n_frames, bool need_feat) {
    const size_t per_stream = (size_t)std::max(n_frames, 1) * kNumChannels * ((clip_fuses(h, n_frames) ? 0 : 4) + (need_feat ? 2 : 0));
    if (per_stream == 0) return h->n_streams;
    size_t t = h->scratch_budget / per_stream;
    if (t < 1) t = 1;
    if (t > (size_t)h->n_streams) t = (size_t)h->n_streams;
    return (int)t;
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
        // size of this particular tile -- the scratch was sized for the fused form)
        ProfScope p(h, 0, st);
        CU(h, launch_frontend_clip_fused(h->P, h->d_carry + (size_t)first * kWindow, h->used, d_audio, audio_stride, n_samples, n, n_frames,
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

// one model step per stream -> the stream-parallel live-step kernels (fp32: mww_nn_live.cuh, int8: mww_nn_i8_live.cuh)
bool use_live(const mww_t *h, int n_rows) { return h->has_nn && !h->generic && n_rows == 3 && !h->no_live; }

// rotate every ring back to the canonical layout before anything that assumes it (clip kernels, mww_get_state)
int canonicalise_rings(mww_t *h, cudaStream_t st) {
    bool any = false;
    for (int i = 0; i < 5; ++i) any = any || h->live_heads.h[i] != 0;
    if (!any || !h->has_nn) return MWW_OK;
    if (h->quantized) CU(h, launch_nn_i8_live_canonicalise(static_cast<int8_t *>(h->d_nn_state), h->n_streams, h->live_heads, st));
    else CU(h, launch_nn_live_canonicalise(static_cast<float *>(h->d_nn_state), h->n_streams, h->live_heads, st));
    h->launches += 1;
    h->live_heads = LiveHeads{};
    return MWW_OK;
}
// once per API call, around the tile loop
int begin_nn_call(mww_t *h, int n_rows, cudaStream_t st) { return use_live(h, n_rows) ? MWW_OK : canonicalise_rings(h, st); }
void end_nn_call(mww_t *h, int n_rows) {
    if (!use_live(h, n_rows)) return;
    for (int i = 0; i < 5; ++i) h->live_heads.h[i] = (h->live_heads.h[i] + 1) % kLiveRingRows[i];
}

int run_nn_tile(mww_t *h, int first, int n, const void *d_rows, int row_type, long long rows_stream_stride_rows, int n_rows,
                float *d_probs, long long probs_stride, cudaStream_t st) {
    ProfScope p(h, 2, st);
    if (h->generic) {
        // any architecture other than the compiled-in one: run-time-geometry kernels (mww_nn_generic.cuh)
        if (row_type != MWW_ROWS_F32 && row_type != MWW_ROWS_U16 && row_type != MWW_ROWS_I8) return fail(h, MWW_EINVAL, "unknown row_type");
        if (row_type == MWW_ROWS_I8 && !h->quantized) return fail(h, MWW_EINVAL, "int8 rows need a quantised model (inference.py:110)");
        const size_t rb = row_type == MWW_ROWS_F32 ? 4 : (row_type == MWW_ROWS_U16 ? 2 : 1);
        const int rt = row_type == MWW_ROWS_U16 ? 0 : (row_type == MWW_ROWS_F32 ? 1 : 2);
        if (h->quantized)
            CU(h, launch_nn_generic_i8(h->G, h->GQ, static_cast<int8_t *>(h->d_nn_state) + (size_t)first * h->state_elems,
                                       static_cast<int8_t *>(h->d_pend) + (size_t)first * h->pend_cap * kNumChannels, h->n_pend, d_rows,
                                       rows_stream_stride_rows * kNumChannels * (long long)rb, n_rows, rt, d_probs, probs_stride, n, st));
        else
            CU(h, launch_nn_generic_f32(h->G, h->GW, static_cast<float *>(h->d_nn_state) + (size_t)first * h->state_elems,
                                        static_cast<float *>(h->d_pend) + (size_t)first * h->pend_cap * kNumChannels, h->n_pend, d_rows,
                                        rows_stream_stride_rows * kNumChannels * (long long)rb, n_rows, rt, d_probs, probs_stride, n, st));
        h->launches += 1;
        return MWW_OK;
    }
    if (h->quantized) {
        if (row_type == MWW_ROWS_F32 || row_type == MWW_ROWS_U16 || row_type == MWW_ROWS_I8) {
            const size_t rb = row_type == MWW_ROWS_F32 ? 4 : (row_type == MWW_ROWS_U16 ? 2 : 1);
            if (reinterpret_cast<uintptr_t>(d_rows) % 16 != 0)          // the integer kernels read rows 8 / 16 bytes at a time
                return fail(h, MWW_EINVAL, "feature rows for an int8 model must be 16-byte aligned");
            if (use_live(h, n_rows)) {
                CU(h, launch_nn_i8_live(h->Wq, static_cast<int8_t *>(h->d_nn_state) + (size_t)first * h->state_elems,
                                        static_cast<int8_t *>(h->d_pend) + (size_t)first * h->pend_cap * kNumChannels, h->n_pend, d_rows,
                                        rows_stream_stride_rows * kNumChannels * (long long)rb, row_type, d_probs, probs_stride, n,
                                        h->live_heads, h->sm_count, st));
                h->launches += 1;
                return MWW_OK;
            }
            CU(h, launch_nn_i8(h->Wq, static_cast<int8_t *>(h->d_nn_state) + (size_t)first * h->state_elems,
                               static_cast<int8_t *>(h->d_pend) + (size_t)first * h->pend_cap * kNumChannels, h->n_pend, d_rows,
                               rows_stream_stride_rows * kNumChannels * (long long)rb, n_rows, row_type, d_probs, probs_stride, n, st));
            h->launches += 1;
            return MWW_OK;
        }
        return fail(h, MWW_EINVAL, "unknown row_type");
    }
    if (row_type == MWW_ROWS_I8) return fail(h, MWW_EINVAL, "int8 rows need a quantised model (inference.py:110)");
    const size_t rb = row_type == MWW_ROWS_F32 ? 4 : 2;
    if (use_live(h, n_rows)) {
        // exactly one model step per stream: the stream-parallel live-step kernel (HBM-bound on the ring state)
        CU(h, launch_nn_f32_live(h->W, static_cast<float *>(h->d_nn_state) + (size_t)first * h->state_elems,
                                 static_cast<float *>(h->d_pend) + (size_t)first * h->pend_cap * kNumChannels, h->n_pend, d_rows,
                                 rows_stream_stride_rows * kNumChannels * (long long)rb, row_type == MWW_ROWS_F32, d_probs, probs_stride, n,
                                 h->live_heads, h->sm_count, h->live_variant, st));
        h->launches += 1;
        return MWW_OK;
    }
    if (!h->no_tc && row_type == MWW_ROWS_U16 && (h->n_pend + n_rows) / 3 >= kTcMinSteps && reinterpret_cast<uintptr_t>(d_rows) % 16 == 0 &&
        (rows_stream_stride_rows * kNumChannels * 2) % 16 == 0) {
        // long calls on raw frontend rows: time is the M dimension of wgmma (mww_nn_tc.cu)
        CU(h, launch_nn_f32_tc(h->W, h->TW, static_cast<float *>(h->d_nn_state) + (size_t)first * h->state_elems,
                               static_cast<float *>(h->d_pend) + (size_t)first * h->pend_cap * kNumChannels, h->n_pend,
                               static_cast<const uint16_t *>(d_rows), rows_stream_stride_rows * kNumChannels, n_rows, d_probs, probs_stride, n,
                               h->sm_count, st));
        h->launches += 1;
        return MWW_OK;
    }
    CU(h, launch_nn_f32(h->W, static_cast<float *>(h->d_nn_state) + (size_t)first * h->state_elems,
                        static_cast<float *>(h->d_pend) + (size_t)first * h->pend_cap * kNumChannels, h->n_pend, d_rows,
                        rows_stream_stride_rows * kNumChannels * (long long)rb, n_rows, row_type == MWW_ROWS_F32, d_probs, probs_stride,
                        nullptr, n, st));
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

struct Need { const char *name; uint32_t dtype; size_t count; };

// weights of an architecture other than the compiled-in one (tensor names and layouts: microwakeword_b200/model_file.py,
// the same names the CPU checker reads)
int upload_weights_generic(mww_t *h, const uint8_t *blob, size_t n, const Tensor &arch) {
    GenArch &G = h->G;
    const int rc_arch = gen_arch_from_tensor(reinterpret_cast<const int32_t *>(arch.data), (int)(arch.nbytes / 4), &G);
    if (rc_arch == -1) return fail(h, MWW_EMODEL, "model container: malformed 'arch' tensor");
    if (rc_arch != 0 || (size_t)G.sm_elems * 4 > 200 * 1024)
        return fail(h, MWW_EUNSUPPORTED, "model container: architecture outside the supported range (first_conv_kernel_size >= stride, <= 8 blocks, "
                                         "<= 512 channels, kernels <= 64 taps, ring buffers of one stream within 200 KB)");
    Tensor probe;
    h->quantized = find_tensor(blob, n, "q/scales", &probe);
    h->generic = true;
    h->stride = G.stride; h->pend_cap = G.pend_cap; h->state_elems = G.state_elems; h->macs_per_step = G.macs_per_step;
    size_t total = 1 << 16;                          // room for alignment padding; tensors are added below
    {
        uint32_t hdr[4];
        memcpy(hdr, blob + 8, 16);
        total += n + (size_t)hdr[1] * 256;
    }
    CU(h, cudaMalloc(&h->d_weights, total));
    size_t cur = 0;
    cudaError_t e = cudaSuccess;
    char name[64];
    auto get = [&](const char *nm, uint32_t dtype, size_t count, const void **dev) -> int {
        Tensor t;
        static const size_t esz[6] = {4, 1, 4, 1, 2, 2};
        if (!find_tensor(blob, n, nm, &t)) return fail(h, MWW_EMODEL, std::string("model container: missing tensor ") + nm);
        if (t.dtype != dtype || t.nbytes != count * esz[dtype]) return fail(h, MWW_EMODEL, std::string("model container: wrong dtype/size for ") + nm);
        if (cur + t.nbytes + 256 > total) return fail(h, MWW_EMODEL, "model container: tensors larger than the container");
        if (!upload(h->d_weights, cur, t.data, (size_t)t.nbytes, reinterpret_cast<const uint8_t **>(dev), &e)) return cuda_fail(h, e, "weight upload");
        return MWW_OK;
    };
    auto scalar = [&](const char *nm, int32_t *out) -> int {
        Tensor t;
        if (!find_tensor(blob, n, nm, &t) || t.nbytes != 4) return fail(h, MWW_EMODEL, std::string("model container: ") + nm);
        memcpy(out, t.data, 4);
        return MWW_OK;
    };
    int rc;
    const size_t k0f = (size_t)G.k0 * kNumChannels * G.c0;
    if (!h->quantized) {
        GenWeightsF32 &W = h->GW;
        if ((rc = get("first_conv/w", 0, k0f, (const void **)&W.w0))) return rc;
        for (int i = 0; i < G.n_blocks; ++i) {
            snprintf(name, sizeof name, "b%d/dw/w", i); if ((rc = get(name, 0, (size_t)G.kmax[i] * G.cin[i], (const void **)&W.dw_w[i]))) return rc;
            snprintf(name, sizeof name, "b%d/dw/b", i); if ((rc = get(name, 0, G.cin[i], (const void **)&W.dw_b[i]))) return rc;
            snprintf(name, sizeof name, "b%d/pw/w", i); if ((rc = get(name, 0, (size_t)G.cin[i] * G.cout[i], (const void **)&W.pw_w[i]))) return rc;
            snprintf(name, sizeof name, "b%d/pw/b", i); if ((rc = get(name, 0, G.cout[i], (const void **)&W.pw_b[i]))) return rc;
        }
        if ((rc = get("head/w", 0, (size_t)G.head_rows * G.c_last, (const void **)&W.head_w))) return rc;
        if ((rc = get("head/b", 0, 1, (const void **)&W.head_b))) return rc;
        return MWW_OK;
    }
    GenWeightsI8 &Q = h->GQ;
    if ((rc = get("q/first_conv/w", 1, k0f, (const void **)&Q.w0))) return rc;
    if ((rc = get("q/first_conv/bias", 2, G.c0, (const void **)&Q.b0))) return rc;
    if ((rc = get("q/first_conv/mult", 2, G.c0, (const void **)&Q.m0))) return rc;
    if ((rc = get("q/first_conv/shift", 2, G.c0, (const void **)&Q.s0))) return rc;
    for (int i = 0; i < G.n_blocks; ++i) {
        snprintf(name, sizeof name, "q/b%d/dw/w", i); if ((rc = get(name, 1, (size_t)G.kmax[i] * G.cin[i], (const void **)&Q.dw_w[i]))) return rc;
        snprintf(name, sizeof name, "q/b%d/dw/bias", i); if ((rc = get(name, 2, G.cin[i], (const void **)&Q.dw_b[i]))) return rc;
        snprintf(name, sizeof name, "q/b%d/dw/mult", i); if ((rc = get(name, 2, G.cin[i], (const void **)&Q.dw_m[i]))) return rc;
        snprintf(name, sizeof name, "q/b%d/dw/shift", i); if ((rc = get(name, 2, G.cin[i], (const void **)&Q.dw_s[i]))) return rc;
        snprintf(name, sizeof name, "q/b%d/pw/w", i); if ((rc = get(name, 1, (size_t)G.cin[i] * G.cout[i], (const void **)&Q.pw_w[i]))) return rc;
        snprintf(name, sizeof name, "q/b%d/pw/bias", i); if ((rc = get(name, 2, G.cout[i], (const void **)&Q.pw_b[i]))) return rc;
        snprintf(name, sizeof name, "q/b%d/pw/mult", i); if ((rc = get(name, 2, G.cout[i], (const void **)&Q.pw_m[i]))) return rc;
        snprintf(name, sizeof name, "q/b%d/pw/shift", i); if ((rc = get(name, 2, G.cout[i], (const void **)&Q.pw_s[i]))) return rc;
    }
    if ((rc = get("q/head/w", 1, (size_t)G.head_rows * G.c_last, (const void **)&Q.head_w))) return rc;
    if ((rc = get("q/logistic_lut", 1, 256, (const void **)&Q.lut))) return rc;
    if ((rc = scalar("q/head/bias", &Q.head_bias)) || (rc = scalar("q/head/mult", &Q.head_mult)) || (rc = scalar("q/head/shift", &Q.head_shift))) return rc;
    const size_t n_q = 4 + 2 * (size_t)G.n_blocks;       // in, first conv, (depthwise, pointwise) per block, logit, prob
    Tensor sc, zp;
    if (!find_tensor(blob, n, "q/scales", &sc) || sc.nbytes != n_q * 4 || !find_tensor(blob, n, "q/zps", &zp) || zp.nbytes != n_q * 4)
        return fail(h, MWW_EMODEL, "model container: q/scales / q/zps must hold 4 + 2 * n_blocks entries");
    std::vector<float> scales(n_q);
    memcpy(scales.data(), sc.data, n_q * 4);
    memcpy(Q.zp, zp.data, n_q * 4);
    Q.in_scale = scales[0];
    h->in_scale = scales[0]; h->in_zp = Q.zp[0];
    h->out_scale = scales[n_q - 1]; h->out_zp = 0;      // uint8 output tensor: zero point -128 + 128 (utils.py:338)
    return MWW_OK;
}

int upload_weights(mww_t *h, const uint8_t *blob, size_t n) {
    Tensor arch;
    if (!find_tensor(blob, n, "arch", &arch) || arch.dtype != 2) return fail(h, MWW_EMODEL, "model container: missing 'arch' tensor or bad magic/version");
    // the tensor-core kernels are compiled for the okay_nabu MixedNet (first conv 32x5 stride 3; MixConv [5],[7,11],[9,15],[23];
    // pointwise 64x4; 17-row head); every other architecture takes the run-time-geometry path.  MWW_FORCE_GENERIC=1 sends
    // okay_nabu through it as well (tests compare the two paths).
    if (arch.nbytes != sizeof kOkayNabuArch || memcmp(arch.data, kOkayNabuArch, sizeof kOkayNabuArch) != 0 || getenv("MWW_FORCE_GENERIC") != nullptr)
        return upload_weights_generic(h, blob, n, arch);
    Tensor probe;
    h->quantized = find_tensor(blob, n, "q/scales", &probe);
    const size_t total = 1 << 20;
    CU(h, cudaMalloc(&h->d_weights, total));
    size_t cur = 0;
    cudaError_t e = cudaSuccess;
    char name[64];
    auto get = [&](const char *nm, uint32_t dtype, size_t count, const void **dev) -> int {
        Tensor t;
        static const size_t esz[6] = {4, 1, 4, 1, 2, 2};
        if (!find_tensor(blob, n, nm, &t)) return fail(h, MWW_EMODEL, std::string("model container: missing tensor ") + nm);
        if (t.dtype != dtype || t.nbytes != count * esz[dtype]) return fail(h, MWW_EMODEL, std::string("model container: wrong dtype/size for ") + nm);
        if (!upload(h->d_weights, cur, t.data, (size_t)t.nbytes, reinterpret_cast<const uint8_t **>(dev), &e)) return cuda_fail(h, e, "weight upload");
        return MWW_OK;
    };
    static const int cin[4] = {32, 64, 64, 64}, kmax[4] = {5, 11, 15, 23};
    int rc;
    if (!h->quantized) {
        if ((rc = get("first_conv/w", 0, 5 * 40 * 32, (const void **)&h->W.w0))) return rc;
        for (int i = 0; i < 4; ++i) {
            snprintf(name, sizeof name, "b%d/dw/w", i); if ((rc = get(name, 0, (size_t)kmax[i] * cin[i], (const void **)&h->W.dw_w[i]))) return rc;
            snprintf(name, sizeof name, "b%d/dw/b", i); if ((rc = get(name, 0, cin[i], (const void **)&h->W.dw_b[i]))) return rc;
            snprintf(name, sizeof name, "b%d/pw/w", i); if ((rc = get(name, 0, (size_t)cin[i] * 64, (const void **)&h->W.pw_w[i]))) return rc;
            snprintf(name, sizeof name, "b%d/pw/b", i); if ((rc = get(name, 0, 64, (const void **)&h->W.pw_b[i]))) return rc;
        }
        if ((rc = get("head/w", 0, 17 * 64, (const void **)&h->W.head_w))) return rc;
        if ((rc = get("head/b", 0, 1, (const void **)&h->W.head_b))) return rc;
        {
            // tensor-core operands: 3xTF32 split + slot layout, once per model (mww_nn_tc.h)
            Tensor tw0, tpw[4];
            bool ok = find_tensor(blob, n, "first_conv/w", &tw0);
            const float *pw_host[4];
            for (int i = 0; i < 4 && ok; ++i) {
                snprintf(name, sizeof name, "b%d/pw/w", i);
                ok = find_tensor(blob, n, name, &tpw[i]);
                pw_host[i] = reinterpret_cast<const float *>(tpw[i].data);
            }
            if (!ok) return fail(h, MWW_EMODEL, "model container: fp32 weights missing");
            std::vector<float> w0_copy(5 * 40 * 32), pw_copy[4];
            memcpy(w0_copy.data(), tw0.data, w0_copy.size() * 4);                    // container tensors are not necessarily 4-byte aligned
            const float *pw_al[4];
            for (int i = 0; i < 4; ++i) {
                pw_copy[i].resize((size_t)cin[i] * 64);
                memcpy(pw_copy[i].data(), pw_host[i], pw_copy[i].size() * 4);
                pw_al[i] = pw_copy[i].data();
            }
            std::vector<unsigned char> tcb;
            size_t offs[5];
            build_tc_weights(w0_copy.data(), pw_al, &tcb, offs);
            const unsigned char *dev_tc = nullptr;
            if (cur + tcb.size() + 256 > total) return fail(h, MWW_EMODEL, "weight arena too small for the tensor-core operands");
            if (!upload(h->d_weights, cur, tcb.data(), tcb.size(), &dev_tc, &e)) return cuda_fail(h, e, "weight upload");
            h->TW.fc = dev_tc + offs[0];
            for (int i = 0; i < 4; ++i) h->TW.pw[i] = dev_tc + offs[1 + i];
        }
    } else {
        NnWeightsI8 &Q = h->Wq;
        if ((rc = get("q/first_conv/w", 1, 5 * 40 * 32, (const void **)&Q.w0))) return rc;
        if ((rc = get("q/first_conv/bias", 2, 32, (const void **)&Q.b0))) return rc;
        if ((rc = get("q/first_conv/mult", 2, 32, (const void **)&Q.m0))) return rc;
        if ((rc = get("q/first_conv/shift", 2, 32, (const void **)&Q.s0))) return rc;
        for (int i = 0; i < 4; ++i) {
            snprintf(name, sizeof name, "q/b%d/dw/w", i); if ((rc = get(name, 1, (size_t)kmax[i] * cin[i], (const void **)&Q.dw_w[i]))) return rc;
            snprintf(name, sizeof name, "q/b%d/dw/bias", i); if ((rc = get(name, 2, cin[i], (const void **)&Q.dw_b[i]))) return rc;
            snprintf(name, sizeof name, "q/b%d/dw/mult", i); if ((rc = get(name, 2, cin[i], (const void **)&Q.dw_m[i]))) return rc;
            snprintf(name, sizeof name, "q/b%d/dw/shift", i); if ((rc = get(name, 2, cin[i], (const void **)&Q.dw_s[i]))) return rc;
            snprintf(name, sizeof name, "q/b%d/pw/w", i); if ((rc = get(name, 1, (size_t)cin[i] * 64, (const void **)&Q.pw_w[i]))) return rc;
            snprintf(name, sizeof name, "q/b%d/pw/bias", i); if ((rc = get(name, 2, 64, (const void **)&Q.pw_b[i]))) return rc;
            snprintf(name, sizeof name, "q/b%d/pw/mult", i); if ((rc = get(name, 2, 64, (const void **)&Q.pw_m[i]))) return rc;
            snprintf(name, sizeof name, "q/b%d/pw/shift", i); if ((rc = get(name, 2, 64, (const void **)&Q.pw_s[i]))) return rc;
        }
        if ((rc = get("q/head/w", 1, 17 * 64, (const void **)&Q.head_w))) return rc;
        if ((rc = get("q/logistic_lut", 1, 256, (const void **)&Q.lut))) return rc;
        Tensor t;
        if (!find_tensor(blob, n, "q/head/bias", &t) || t.nbytes != 4) return fail(h, MWW_EMODEL, "model container: q/head/bias");
        memcpy(&Q.head_bias, t.data, 4);
        if (!find_tensor(blob, n, "q/head/mult", &t) || t.nbytes != 4) return fail(h, MWW_EMODEL, "model container: q/head/mult");
        memcpy(&Q.head_mult, t.data, 4);
        if (!find_tensor(blob, n, "q/head/shift", &t) || t.nbytes != 4) return fail(h, MWW_EMODEL, "model container: q/head/shift");
        memcpy(&Q.head_shift, t.data, 4);
        Tensor sc, zp;
        if (!find_tensor(blob, n, "q/scales", &sc) || sc.nbytes != 12 * 4 || !find_tensor(blob, n, "q/zps", &zp) || zp.nbytes != 12 * 4)
            return fail(h, MWW_EMODEL, "model container: q/scales / q/zps must hold 12 entries");
        float scales[12];
        memcpy(scales, sc.data, sizeof scales);
        memcpy(Q.zp, zp.data, sizeof Q.zp);
        Q.in_scale = scales[0];
        h->in_scale = scales[0]; h->in_zp = Q.zp[0];
        // tensor-core operands: K-contiguous weight rows and zero-point-folded biases (mww_nn_i8_prep.h)
        {
            Tensor tw0, tb0, tpw[4], tpb[4];
            bool ok = find_tensor(blob, n, "q/first_conv/w", &tw0) && find_tensor(blob, n, "q/first_conv/bias", &tb0);
            const int8_t *pw_w[4]; const int32_t *pw_b[4];
            for (int i = 0; i < 4 && ok; ++i) {
                snprintf(name, sizeof name, "q/b%d/pw/w", i); ok = ok && find_tensor(blob, n, name, &tpw[i]);
                snprintf(name, sizeof name, "q/b%d/pw/bias", i); ok = ok && find_tensor(blob, n, name, &tpb[i]);
                pw_w[i] = reinterpret_cast<const int8_t *>(tpw[i].data); pw_b[i] = reinterpret_cast<const int32_t *>(tpb[i].data);
            }
            if (!ok) return fail(h, MWW_EMODEL, "model container: int8 weights missing");
            I8MmaOperands ops;
            build_i8_mma_operands(reinterpret_cast<const int8_t *>(tw0.data), reinterpret_cast<const int32_t *>(tb0.data), pw_w, pw_b, Q.zp, &ops);
            bool up = upload(h->d_weights, cur, ops.w0t.data(), ops.w0t.size(), &Q.w0t, &e) &&
                      upload(h->d_weights, cur, ops.b0f.data(), ops.b0f.size() * 4, &Q.b0f, &e);
            for (int i = 0; i < 4 && up; ++i)
                up = upload(h->d_weights, cur, ops.pwt[i].data(), ops.pwt[i].size(), &Q.pwt[i], &e) &&
                     upload(h->d_weights, cur, ops.pw_bf[i].data(), ops.pw_bf[i].size() * 4, &Q.pw_bf[i], &e);
            if (!up) return cuda_fail(h, e, "weight upload");
            if (getenv("MWW_NO_QLUT") == nullptr) {
                std::vector<int8_t> qlut;
                build_feature_qlut(Q.in_scale, Q.zp[0], &qlut);
                if (!upload(h->d_weights, cur, qlut.data(), qlut.size(), &Q.qlut, &e)) return cuda_fail(h, e, "weight upload");
            }
        }
        h->out_scale = scales[11]; h->out_zp = 0;   // uint8 output tensor: zero point -128 + 128 (utils.py:338)
    }
    return MWW_OK;
}

int zero_state(mww_t *h, cudaStream_t st) {
    const size_t S = (size_t)h->n_streams;
    CU(h, cudaMemsetAsync(h->d_carry, 0, S * kWindow * sizeof(int16_t), st));
    CU(h, cudaMemsetAsync(h->d_estimate, 0, S * kNumChannels * sizeof(uint32_t), st));
    h->used = 0;
    h->n_pend = 0;
    if (!h->has_nn) return MWW_OK;
    if (h->quantized && h->generic) {
        CU(h, launch_gen_fill_state_i8(h->G, h->GQ, static_cast<int8_t *>(h->d_nn_state), static_cast<int8_t *>(h->d_pend), h->n_streams, nullptr, h->n_streams, st));
        h->launches += 1;
    } else if (h->quantized) {
        CU(h, launch_fill_state_i8(h->Wq, static_cast<int8_t *>(h->d_nn_state), static_cast<int8_t *>(h->d_pend), nullptr, h->n_streams, h->n_streams, st));
        h->launches += 1;
    } else {
        CU(h, cudaMemsetAsync(h->d_nn_state, 0, S * h->state_elems * 4, st));
        CU(h, cudaMemsetAsync(h->d_pend, 0, S * h->pend_cap * kNumChannels * 4, st));
    }
    h->live_heads = LiveHeads{};
    h->used = 0;
    h->n_pend = 0;
    return MWW_OK;
}

void destroy_impl(mww_t *h) {
    if (!h) return;
    DeviceGuard guard(h->device);
    cudaFree(h->d_tables); cudaFree(h->d_weights); cudaFree(h->d_carry); cudaFree(h->d_estimate);
    cudaFree(h->d_nn_state); cudaFree(h->d_pend); cudaFree(h->d_v); cudaFree(h->d_feat); cudaFree(h->d_ids);
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
    if (n_samples < 0 || (n_samples > 0 && !d_audio) || audio_stride < n_samples) return fail(h, MWW_EINVAL, std::string(who) + ": bad audio arguments");
    ENTER_STATEFUL(h);
    cudaStream_t st = static_cast<cudaStream_t>(cu_stream);
    const int n_frames = frames_for(h, n_samples);
    if (n_frames > max_rows || (n_frames > 0 && !d_feat))
        return fail(h, MWW_EINVAL, std::string(who) + ": feature buffer too small for the rows this call emits");
    const int tile = tile_streams(h, n_frames, false);
    int rc = ensure_scratch(h, v_scratch_bytes(h, tile, n_frames), 0);
    if (rc) return rc;
    for (int first = 0; first < h->n_streams; first += tile) {
        const int n = std::min(tile, h->n_streams - first);
        rc = run_frontend_tile(h, first, n, d_audio + (size_t)first * audio_stride, audio_stride, n_samples, n_frames,
                               d_feat + (size_t)first * max_rows * kNumChannels, (long long)max_rows * kNumChannels, st);
        if (rc) return rc;
    }
    if (n_samples > 0) {
        rc = run_carry_tile(h, 0, h->n_streams, d_audio, audio_stride, n_samples, n_frames, st);
        if (rc) return rc;
    }
    h->used = h->used + n_samples - n_frames * h->hop;
    if (h_rows_out) *h_rows_out = n_frames;
    return MWW_OK;
}

// mww_predict_clip / mww_predict_clip_f32
template <typename T>
int predict_clip_impl(mww_t *h, const char *who, const T *d_audio, int n_samples, long long audio_stride, float *d_probs, int max_probs,
                      int *h_probs_out, void *cu_stream) {
    if (!h) return MWW_EINVAL;
    if (n_samples < 0 || (n_samples > 0 && !d_audio) || audio_stride < n_samples) return fail(h, MWW_EINVAL, std::string(who) + ": bad audio arguments");
    if (!h->has_nn) return fail(h, MWW_EINVAL, std::string(who) + ": frontend-only handle (created without a model)");
    ENTER_STATEFUL(h);
    cudaStream_t st = static_cast<cudaStream_t>(cu_stream);
    const int n_frames = frames_for(h, n_samples);
    const int n_steps = (h->n_pend + n_frames) / h->stride;
    if (n_steps > max_probs || (n_steps > 0 && !d_probs)) return fail(h, MWW_EINVAL, std::string(who) + ": probability buffer too small");
    const int tile = tile_streams(h, n_frames, true);
    int rc = ensure_scratch(h, v_scratch_bytes(h, tile, n_frames), (size_t)tile * std::max(n_frames, 1) * kNumChannels * 2);
    if (rc) return rc;
    rc = begin_nn_call(h, n_frames, st);
    if (rc) return rc;
    for (int first = 0; first < h->n_streams; first += tile) {
        const int n = std::min(tile, h->n_streams - first);
        rc = run_frontend_tile(h, first, n, d_audio + (size_t)first * audio_stride, audio_stride, n_samples, n_frames, h->d_feat,
                               (long long)n_frames * kNumChannels, st);
        if (rc) return rc;
        rc = run_nn_tile(h, first, n, h->d_feat, MWW_ROWS_U16, n_frames, n_frames, d_probs + (size_t)first * max_probs, max_probs, st);
        if (rc) return rc;
    }
    end_nn_call(h, n_frames);
    if (n_samples > 0) {
        rc = run_carry_tile(h, 0, h->n_streams, d_audio, audio_stride, n_samples, n_frames, st);
        if (rc) return rc;
    }
    h->used = h->used + n_samples - n_frames * h->hop;
    h->n_pend = (h->n_pend + n_frames) % h->stride;
    if (h_probs_out) *h_probs_out = n_steps;
    return MWW_OK;
}

}  // namespace

extern "C" {

int mww_create(const void *model_blob, size_t n_bytes, int device, int n_streams, mww_t **out) {
    if (out) *out = nullptr;
    if (!out || n_streams < 1) return fail(nullptr, MWW_EINVAL, "mww_create: bad arguments");
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0)
        return fail(nullptr, MWW_ECUDA, std::string("no CUDA device available (this library has no CPU fallback): ") + cudaGetErrorString(e));
    if (device < 0 || device >= count) return fail(nullptr, MWW_EINVAL, "mww_create: device index out of range");
    DeviceGuard guard(device);
    if (guard.err != cudaSuccess) return cuda_fail(nullptr, guard.err, "cudaSetDevice");
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
    h->has_nn = model_blob != nullptr;
    if (h->has_nn) {
        uint64_t x = 1469598103934665603ull;
        for (size_t i = 0; i < n_bytes; ++i) x = (x ^ static_cast<const uint8_t *>(model_blob)[i]) * 1099511628211ull;
        h->model_hash = x;
    }
    int rc = upload_tables(h);
    if (rc == MWW_OK && h->has_nn) rc = upload_weights(h, static_cast<const uint8_t *>(model_blob), n_bytes);
    if (rc == MWW_OK) {
        const size_t S = (size_t)n_streams;
        cudaError_t a = cudaMalloc(&h->d_carry, S * kWindow * sizeof(int16_t));
        if (a == cudaSuccess) a = cudaMalloc(&h->d_estimate, S * kNumChannels * sizeof(uint32_t));
        if (a == cudaSuccess && h->has_nn) a = cudaMalloc(&h->d_nn_state, S * h->state_elems * elem_size(h));
        if (a == cudaSuccess && h->has_nn) a = cudaMalloc(&h->d_pend, S * h->pend_cap * kNumChannels * elem_size(h));
        if (a != cudaSuccess) rc = fail(h, a == cudaErrorMemoryAllocation ? MWW_ENOMEM : MWW_ECUDA, std::string("state allocation: ") + cudaGetErrorString(a));
    }
    if (rc == MWW_OK) rc = zero_state(h, nullptr);
    if (rc == MWW_OK) { cudaError_t s = cudaDeviceSynchronize(); if (s != cudaSuccess) rc = cuda_fail(h, s, "cudaDeviceSynchronize"); }
    if (rc != MWW_OK) { g_create_error = h->err; destroy_impl(h); return rc; }
    *out = h;
    return MWW_OK;
}

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

int mww_get_info(const mww_t *h, mww_info *o) {
    if (!h || !o) return MWW_EINVAL;
    memset(o, 0, sizeof *o);
    o->n_streams = h->n_streams; o->device = h->device; o->is_quantized = h->quantized;
    o->input_feature_slices = h->stride; o->num_features = kNumChannels;
    o->input_scale = h->in_scale; o->input_zero_point = h->in_zp;
    o->output_scale = h->out_scale; o->output_zero_point = h->out_zp;
    o->state_bytes_per_stream = (int)(h->state_elems * elem_size(h));
    o->frontend_buffered = h->used; o->pending_rows = h->n_pend;
    o->sm_count = h->sm_count; o->macs_per_step = (int)h->macs_per_step;
    o->hop_samples = h->hop;
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

int fill_by_id(mww_t *h, void *base, size_t bytes_per_stream, const int32_t *d_ids, int n, cudaStream_t st) {
    const long long words = (long long)(bytes_per_stream / 4);
    const long long total = words * n;
    if (total <= 0) return MWW_OK;
    const unsigned blocks = (unsigned)std::min<long long>((total + 255) / 256, (long long)h->sm_count * 16);
    fill_by_id_kernel<<<blocks, 256, 0, st>>>(static_cast<uint32_t *>(base), words, 0u, d_ids, n, h->n_streams);
    CU(h, cudaGetLastError());
    h->launches += 1;
    return MWW_OK;
}

// fresh state for the listed streams: a handful of launches whatever the length of the list
int reset_by_id(mww_t *h, const int32_t *d_ids, int n, cudaStream_t st) {
    if (n <= 0) return MWW_OK;
    int rc = fill_by_id(h, h->d_carry, kWindow * sizeof(int16_t), d_ids, n, st);
    if (rc == MWW_OK) rc = fill_by_id(h, h->d_estimate, kNumChannels * sizeof(uint32_t), d_ids, n, st);
    if (rc != MWW_OK || !h->has_nn) return rc;
    if (h->quantized && h->generic) {
        CU(h, launch_gen_fill_state_i8(h->G, h->GQ, static_cast<int8_t *>(h->d_nn_state), static_cast<int8_t *>(h->d_pend), n, d_ids, h->n_streams, st));
        h->launches += 1;
    } else if (h->quantized) {
        CU(h, launch_fill_state_i8(h->Wq, static_cast<int8_t *>(h->d_nn_state), static_cast<int8_t *>(h->d_pend), d_ids, n, h->n_streams, st));
        h->launches += 1;
    } else {
        // zero rings are rotation-invariant, so streams of a handle whose rings are rotated (live mode) can be reset in place
        rc = fill_by_id(h, h->d_nn_state, (size_t)h->state_elems * 4, d_ids, n, st);
        if (rc == MWW_OK) rc = fill_by_id(h, h->d_pend, (size_t)h->pend_cap * kNumChannels * 4, d_ids, n, st);
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
    if ((size_t)n > h->ids_cap) {
        if (h->d_ids) { CU(h, cudaStreamSynchronize(st)); cudaFree(h->d_ids); h->d_ids = nullptr; h->ids_cap = 0; }
        const size_t cap = std::max<size_t>((size_t)n, 1024);
        CU(h, cudaMalloc(&h->d_ids, cap * sizeof(int32_t)));
        h->ids_cap = cap;
    }
    CU(h, cudaMemcpyAsync(h->d_ids, h_ids, (size_t)n * sizeof(int32_t), cudaMemcpyHostToDevice, st));
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
    cudaStream_t st = static_cast<cudaStream_t>(cu_stream);
    const size_t S = (size_t)h->n_streams;
    CU(h, cudaMemsetAsync(h->d_carry, 0, S * kWindow * sizeof(int16_t), st));
    CU(h, cudaMemsetAsync(h->d_estimate, 0, S * kNumChannels * sizeof(uint32_t), st));
    h->used = 0;
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
    return predict_clip_impl(h, "mww_predict_clip", d_audio, n_samples, audio_stride, d_probs, max_probs, h_probs_out, cu_stream);
}
int mww_predict_clip_f32(mww_t *h, const float *d_audio, int n_samples, long long audio_stride, float *d_probs, int max_probs,
                         int *h_probs_out, void *cu_stream) {
    return predict_clip_impl(h, "mww_predict_clip_f32", d_audio, n_samples, audio_stride, d_probs, max_probs, h_probs_out, cu_stream);
}

int mww_infer_features(mww_t *h, const void *d_rows, int row_type, int n_rows, long long rows_stride, float *d_probs,
                       int max_probs, int *h_probs_out, void *cu_stream) {
    if (!h) return MWW_EINVAL;
    if (n_rows < 0 || (n_rows > 0 && !d_rows) || rows_stride < n_rows) return fail(h, MWW_EINVAL, "mww_infer_features: bad row arguments");
    if (row_type < 0 || row_type > 2) return fail(h, MWW_EINVAL, "mww_infer_features: unknown row_type");
    if (!h->has_nn) return fail(h, MWW_EINVAL, "mww_infer_features: frontend-only handle (created without a model)");
    ENTER_STATEFUL(h);
    const int n_steps = (h->n_pend + n_rows) / h->stride;
    if (n_steps > max_probs || (n_steps > 0 && !d_probs)) return fail(h, MWW_EINVAL, "mww_infer_features: probability buffer too small");
    int rc = begin_nn_call(h, n_rows, static_cast<cudaStream_t>(cu_stream));
    if (rc) return rc;
    rc = run_nn_tile(h, 0, h->n_streams, d_rows, row_type, rows_stride, n_rows, d_probs, max_probs, static_cast<cudaStream_t>(cu_stream));
    if (rc == MWW_OK) end_nn_call(h, n_rows);
    if (rc) return rc;
    h->n_pend = (h->n_pend + n_rows) % h->stride;
    if (h_probs_out) *h_probs_out = n_steps;
    return MWW_OK;
}

// ---- staged path: the audio does not live on this GPU ------------------------------------------------------------
// Shared by mww_predict_clip_host (source = host memory, destination = host memory) and mww_predict_clip_remote (source =
// host memory or device memory of a PEER GPU mapped into this process, destination = this GPU).  The streams are cut into
// tiles; a copy stream brings tile t+1 into one of two staging buffers (cudaMemcpyAsync, cudaMemcpyDefault: the copy
// engine of THIS GPU pulls over PCIe or NVLink, no SM is involved on either side) while the kernels of tile t run on the
// compute stream, and for a host destination a third stream drains the scores.
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
int staged_tiles(mww_t *h, const int16_t *src, int n_samples, long long audio_stride, float *dst, int max_probs, bool dst_is_host,
                 int tile, int n_frames, int n_steps) {
    int it = 0;
    for (int first = 0; first < h->n_streams; first += tile, ++it) {
        const int n = std::min(tile, h->n_streams - first);
        const int b = it & 1;
        // the staging buffer is free once the kernels of the tile that used it two iterations ago are done
        if (it >= 2) CU(h, cudaStreamWaitEvent(h->st_h2d, h->ev_compute[b], 0));
        cudaEvent_t tl[4] = {nullptr, nullptr, nullptr, nullptr};
        if (h->profiling) {
            for (int i = 0; i < 4; ++i) { CU(h, cudaEventCreate(&tl[i])); h->tl_ev.push_back(tl[i]); }
            CU(h, cudaEventRecord(tl[0], h->st_h2d));
        }
        if (n_samples > 0) {
            const int16_t *from = src + (size_t)first * audio_stride;
            if (audio_stride == n_samples)       // contiguous block: one linear DMA
                CU(h, cudaMemcpyAsync(h->d_audio_tile[b], from, (size_t)n * n_samples * 2, cudaMemcpyDefault, h->st_h2d));
            else
                CU(h, cudaMemcpy2DAsync(h->d_audio_tile[b], (size_t)n_samples * 2, from, (size_t)audio_stride * 2, (size_t)n_samples * 2, n,
                                        cudaMemcpyDefault, h->st_h2d));
        }
        if (tl[1]) CU(h, cudaEventRecord(tl[1], h->st_h2d));
        CU(h, cudaEventRecord(h->ev_h2d[b], h->st_h2d));
        CU(h, cudaStreamWaitEvent(h->st_compute, h->ev_h2d[b], 0));
        if (tl[2]) CU(h, cudaEventRecord(tl[2], h->st_compute));
        if (dst_is_host && it >= 2) CU(h, cudaStreamWaitEvent(h->st_compute, h->ev_d2h[b], 0));   // score staging buffer drained
        int rc = run_frontend_tile(h, first, n, h->d_audio_tile[b], n_samples, n_samples, n_frames, h->d_feat, (long long)n_frames * kNumChannels, h->st_compute);
        if (rc) return rc;
        float *tile_probs = dst_is_host ? h->d_probs_tile[b] : dst + (size_t)first * max_probs;
        const long long tile_probs_stride = dst_is_host ? std::max(n_steps, 1) : max_probs;
        rc = run_nn_tile(h, first, n, h->d_feat, MWW_ROWS_U16, n_frames, n_frames, tile_probs, tile_probs_stride, h->st_compute);
        if (rc) return rc;
        if (n_samples > 0) {
            rc = run_carry_tile(h, first, n, h->d_audio_tile[b], n_samples, n_samples, n_frames, h->st_compute);
            if (rc) return rc;
        }
        if (tl[3]) CU(h, cudaEventRecord(tl[3], h->st_compute));
        CU(h, cudaEventRecord(h->ev_compute[b], h->st_compute));
        if (dst_is_host) {
            CU(h, cudaStreamWaitEvent(h->st_d2h, h->ev_compute[b], 0));
            if (n_steps > 0)
                CU(h, cudaMemcpy2DAsync(dst + (size_t)first * max_probs, (size_t)max_probs * 4, h->d_probs_tile[b], (size_t)std::max(n_steps, 1) * 4,
                                        (size_t)n_steps * 4, n, cudaMemcpyDeviceToHost, h->st_d2h));
            CU(h, cudaEventRecord(h->ev_d2h[b], h->st_d2h));
        }
    }
    return MWW_OK;
}

// `caller` != nullptr-or-legacy semantics: the call is ordered after everything queued on `caller` so far, and `caller`
// is made to wait for the call's last kernel (asynchronous variant).  host_sync: return only when dst is complete.
int predict_clip_staged(mww_t *h, const char *who, const int16_t *src, int n_samples, long long audio_stride, float *dst, int max_probs,
                        int *h_probs_out, bool dst_is_host, int want_tiles, cudaStream_t caller, bool host_sync) {
    const int n_frames = frames_for(h, n_samples);
    const int n_steps = (h->n_pend + n_frames) / h->stride;
    if (n_steps > max_probs || (n_steps > 0 && !dst)) return fail(h, MWW_EINVAL, std::string(who) + ": probability buffer too small");
    int rc = ensure_pipeline(h);
    if (rc) return rc;
    // tile so that copies and kernels of neighbouring tiles overlap: 16 tiles by default when there are enough streams (the
    // first tile's copy and the last tile's kernels are the only parts that cannot hide behind each other), but never
    // fewer than 2 048 streams per tile so that every launch still fills the GPU
    if (want_tiles <= 0) want_tiles = 16;
    int tile = tile_streams(h, n_frames, true);
    tile = std::max(1, std::min(tile, std::max((h->n_streams + want_tiles - 1) / want_tiles, std::min(h->n_streams, h->min_tile_streams))));
    rc = ensure_scratch(h, v_scratch_bytes(h, tile, n_frames), (size_t)tile * std::max(n_frames, 1) * kNumChannels * 2);
    if (rc) return rc;
    const size_t a_bytes = (size_t)tile * std::max(n_samples, 1) * sizeof(int16_t);
    const size_t p_bytes = dst_is_host ? (size_t)tile * std::max(n_steps, 1) * sizeof(float) : 0;
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
    rc = begin_nn_call(h, n_frames, h->st_compute);
    if (rc == MWW_OK) {
        h->staged_used = true;
        rc = staged_tiles(h, src, n_samples, audio_stride, dst, max_probs, dst_is_host, tile, n_frames, n_steps);
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
    end_nn_call(h, n_frames);
    h->used = h->used + n_samples - n_frames * h->hop;
    h->n_pend = (h->n_pend + n_frames) % h->stride;
    if (h_probs_out) *h_probs_out = n_steps;
    return MWW_OK;
}

}  // namespace

int mww_predict_clip_host(mww_t *h, const int16_t *h_audio, int n_samples, long long audio_stride, float *h_probs, int max_probs,
                          int *h_probs_out) {
    if (!h) return MWW_EINVAL;
    if (n_samples < 0 || (n_samples > 0 && !h_audio) || audio_stride < n_samples) return fail(h, MWW_EINVAL, "mww_predict_clip_host: bad audio arguments");
    if (!h->has_nn) return fail(h, MWW_EINVAL, "mww_predict_clip_host: frontend-only handle (created without a model)");
    ENTER_STATEFUL(h);
    // The call has no stream argument, so it cannot be ordered after one particular stream: it waits for everything the
    // device has been given so far (mww_reset / live calls queued on any stream touch the same per-stream state).
    CU(h, cudaDeviceSynchronize());
    return predict_clip_staged(h, "mww_predict_clip_host", h_audio, n_samples, audio_stride, h_probs, max_probs, h_probs_out, true, 0, nullptr, true);
}

int mww_predict_clip_remote(mww_t *h, const int16_t *src_audio, int n_samples, long long audio_stride, float *d_probs, int max_probs,
                            int *h_probs_out, int n_tiles, void *cu_stream) {
    if (!h) return MWW_EINVAL;
    if (n_samples < 0 || (n_samples > 0 && !src_audio) || audio_stride < n_samples) return fail(h, MWW_EINVAL, "mww_predict_clip_remote: bad audio arguments");
    if (!h->has_nn) return fail(h, MWW_EINVAL, "mww_predict_clip_remote: frontend-only handle (created without a model)");
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
    if (local && n_tiles <= 0) return mww_predict_clip(h, src_audio, n_samples, audio_stride, d_probs, max_probs, h_probs_out, cu_stream);
    ENTER_STATEFUL(h);
    return predict_clip_staged(h, "mww_predict_clip_remote", src_audio, n_samples, audio_stride, d_probs, max_probs, h_probs_out, false, n_tiles,
                               static_cast<cudaStream_t>(cu_stream), false);
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

int mww_get_state(mww_t *h, int16_t *h_carry, uint32_t *h_estimate, void *h_nn, void *h_pending) {
    if (!h) return MWW_EINVAL;
    ENTER_STATEFUL(h);
    CU(h, cudaDeviceSynchronize());
    if (h_nn) {                                    // the exported layout is always the canonical oldest-first one
        const int rc = canonicalise_rings(h, nullptr);
        if (rc) return rc;
        CU(h, cudaDeviceSynchronize());
    }
    const size_t S = (size_t)h->n_streams;
    if (h_carry) CU(h, cudaMemcpy(h_carry, h->d_carry, S * kWindow * 2, cudaMemcpyDeviceToHost));
    if (h_estimate) CU(h, cudaMemcpy(h_estimate, h->d_estimate, S * kNumChannels * 4, cudaMemcpyDeviceToHost));
    if ((h_nn || h_pending) && !h->has_nn) return fail(h, MWW_EINVAL, "frontend-only handle has no NN state");
    if (h_nn) CU(h, cudaMemcpy(h_nn, h->d_nn_state, S * h->state_elems * elem_size(h), cudaMemcpyDeviceToHost));
    if (h_pending) CU(h, cudaMemcpy(h_pending, h->d_pend, S * h->pend_cap * kNumChannels * elem_size(h), cudaMemcpyDeviceToHost));
    return MWW_OK;
}

int mww_set_state(mww_t *h, const int16_t *h_carry, int frontend_buffered, const uint32_t *h_estimate, const void *h_nn,
                  const void *h_pending, int pending_rows) {
    if (!h) return MWW_EINVAL;
    if (frontend_buffered < 0 || frontend_buffered >= kWindow || pending_rows < 0 || pending_rows > h->stride - 1)
        return fail(h, MWW_EINVAL, "mww_set_state: counters out of range");
    ENTER(h);
    CU(h, cudaDeviceSynchronize());
    const size_t S = (size_t)h->n_streams;
    if (h_carry) CU(h, cudaMemcpy(h->d_carry, h_carry, S * kWindow * 2, cudaMemcpyHostToDevice));
    if (h_estimate) CU(h, cudaMemcpy(h->d_estimate, h_estimate, S * kNumChannels * 4, cudaMemcpyHostToDevice));
    if ((h_nn || h_pending) && !h->has_nn) return fail(h, MWW_EINVAL, "frontend-only handle has no NN state");
    if (h_nn) {
        CU(h, cudaMemcpy(h->d_nn_state, h_nn, S * h->state_elems * elem_size(h), cudaMemcpyHostToDevice));
        h->live_heads = LiveHeads{};
    }
    if (h_pending) CU(h, cudaMemcpy(h->d_pend, h_pending, S * h->pend_cap * kNumChannels * elem_size(h), cudaMemcpyHostToDevice));
    h->used = frontend_buffered;
    h->n_pend = pending_rows;
    return MWW_OK;
}

int mww_copy_nn_state(mww_t *dst, const int32_t *h_dst_ids, const mww_t *src_c, const int32_t *h_src_ids, int n, void *cu_stream) {
    if (!dst) return MWW_EINVAL;
    // canonicalising the source's rings changes their layout, not the state they hold
    mww_t *src = const_cast<mww_t *>(src_c);
    if (!src || n < 0 || (n > 0 && (!h_dst_ids || !h_src_ids))) return fail(dst, MWW_EINVAL, "mww_copy_nn_state: bad arguments");
    if (src->device != dst->device) return fail(dst, MWW_EINVAL, "mww_copy_nn_state: the handles are on different devices");
    if (!src->has_nn || !dst->has_nn) return fail(dst, MWW_EINVAL, "mww_copy_nn_state: frontend-only handle has no NN state");
    if (src->model_hash != dst->model_hash || src->quantized != dst->quantized || src->state_elems != dst->state_elems)
        return fail(dst, MWW_EINVAL, "mww_copy_nn_state: the handles were created from different models");
    if (src->n_pend != 0 || dst->n_pend != 0) return fail(dst, MWW_EINVAL, "mww_copy_nn_state: a handle holds pending rows");
    for (int i = 0; i < n; ++i)
        if (h_dst_ids[i] < 0 || h_dst_ids[i] >= dst->n_streams || h_src_ids[i] < 0 || h_src_ids[i] >= src->n_streams)
            return fail(dst, MWW_EINVAL, "mww_copy_nn_state: stream id out of range");
    ENTER_STATEFUL(dst);
    if (src->poisoned) return fail(dst, MWW_ECUDA, "mww_copy_nn_state: the source handle needs mww_reset(h, NULL, 0, stream)");
    cudaStream_t st = static_cast<cudaStream_t>(cu_stream);
    int rc = canonicalise_rings(src, st);
    if (rc) return fail(dst, rc, "mww_copy_nn_state: " + src->err);
    if (dst != src && (rc = canonicalise_rings(dst, st)) != MWW_OK) return rc;
    const size_t bytes = (size_t)dst->state_elems * elem_size(dst);
    char *d = static_cast<char *>(dst->d_nn_state);
    const char *s = static_cast<const char *>(src->d_nn_state);
    for (int i = 0; i < n; ++i) {
        if (dst == src && h_dst_ids[i] == h_src_ids[i]) continue;     // same bytes: nothing to copy (and memcpy needs disjoint ranges)
        CU(dst, cudaMemcpyAsync(d + (size_t)h_dst_ids[i] * bytes, s + (size_t)h_src_ids[i] * bytes, bytes, cudaMemcpyDeviceToDevice, st));
    }
    return MWW_OK;
}

}  // extern "C"
