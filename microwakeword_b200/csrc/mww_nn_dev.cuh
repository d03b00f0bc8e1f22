// mww_nn_dev.cuh -- streaming MixedNet (fp32), time-parallel "clip" formulation, per-thread phases.
//
// Replaces what tf.lite.Interpreter.invoke() executes per 30 ms step at
// microwakeword/inference.py:113-119, i.e. the streaming graph of microwakeword/mixednet.py:307-386
// (first strided conv, four MixConv blocks = ring-buffered grouped depthwise conv + 1x1 pointwise
// with folded BatchNorm + ReLU, 17-row ring, Flatten, Dense(1), sigmoid) with the ring semantics of
// microwakeword/layers/stream.py:581-595.
//
// Hopper-first design: every conv in the graph is a causal 'valid' FIR along time, so a whole chunk of
// TT model steps of one stream is evaluated layer by layer as small dense problems whose M dimension
// is TIME (README.md:27-28 equivalence; the ring state supplies the k-1 rows of history).  The ring
// buffers live in shared memory for the entire clip and touch HBM once per call, instead of the
// reference's 4 176-element state shuffle on every step (stream.py:586-590).
//
// One CTA = one stream, 288 threads, chunks of 36 model steps (1 s of audio = 34 steps = one chunk).
// Shared-memory activation layout is channel-major [c][LD] with time contiguous; columns [0, R) hold the
// ring history, columns [R, R+TT) the chunk's new outputs.  LD is odd, so the depthwise stage -- one lane per
// channel sliding along time -- reads without bank conflicts.  The depthwise output D[c][t] (the A operand
// of the 1x1 contraction) and the 1x1 weights staged in shared memory feed warp-level tensor-core MMAs
// (mww_nn_mma.cuh); their pitches (40 and 72 floats) make the fragment loads bank-conflict free.
// Feature rows are de-interleaved into three planes by (row mod 3) so that the stride-3 first conv reads
// consecutive time steps from consecutive addresses; its K = 200 contraction is split over three warp groups
// whose partial sums meet in shared memory.
#pragma once

#include "mww_common.h"

#if !defined(__CUDA_ARCH__)
#include <math.h>
#endif

namespace mww {

constexpr int kNnThreads = 288;
constexpr int kTT = 36;            // model steps per chunk

struct NnLayerGeom { int cin, kmax, ring, hp, ld, off; };   // off: float offset of the buffer in smem

// geometry of the five ring-carrying activation buffers: inputs of block 0..3 and of the head
// (okay_nabu MixedNet, notebooks/basic_training_notebook.ipynb:503-509; SURVEY.md Appendix A)
constexpr NnLayerGeom kGeom[5] = {
    {32, 5, 4, 4, 41, 0},
    {64, 11, 10, 10, 47, 32 * 41},
    {64, 15, 14, 14, 51, 32 * 41 + 64 * 47},
    {64, 23, 22, 22, 59, 32 * 41 + 64 * 47 + 64 * 51},
    {64, 17, 16, 16, 53, 32 * 41 + 64 * 47 + 64 * 51 + 64 * 59},
};
constexpr int kXFloats = 32 * 41 + 64 * (47 + 51 + 59 + 53);   // 14752
constexpr int kDLd = 40;                                      // 40 = 8 (mod 32): conflict-free mma A fragments
constexpr int kDFloats = 64 * kDLd + 8;                       // + slack: the last m-tile reads 12 rows past kTT
// D[c][t] is WRITTEN with lanes = channels (bank = 8 c + t: 4 banks, 8-way replays) and READ as mma A fragments with
// lanes = (4 channels x 8 steps).  XOR-ing the step with bits 2..4 of the channel keeps a fragment's 8 steps inside
// their aligned 8-block (reads stay conflict-free) and spreads 32 consecutive channels over all 32 banks on the write.
MWW_HD int nn_d_swz(int c) { return (c >> 2) & 7; }
MWW_HD int nn_d_index(int c, int t) { return c * kDLd + (t ^ nn_d_swz(c)); }
constexpr int kUS = 40;                                       // pitch of a feature plane row (u index)
constexpr int kFeatFloats = 3 * kNumChannels * kUS;           // 4800 >= 64*64 staged 1x1 weights
constexpr int kWLdDev = 72;                                   // pitch of staged 1x1 weights (see mww_nn_mma.cuh)
constexpr int kWBFloats = 64 * kWLdDev;                       // second staging buffer for the 1x1 weights
constexpr int kNnSmemFloats = kXFloats + kDFloats + kFeatFloats + kWBFloats;
constexpr int kNnSmemBytes = kNnSmemFloats * 4;               // 103.8 KB -> 2 CTAs / SM
static_assert(kXFloats % 4 == 0 && kDFloats % 4 == 0 && kFeatFloats >= 64 * 72, "smem carve-up");

// per-stream state layout in HBM (floats), oldest row first, [row][channel] -- identical to the oracle
constexpr int kStateOff[6] = {0, 80, 80 + 128, 80 + 128 + 640, 80 + 128 + 640 + 896, 80 + 128 + 640 + 896 + 1408};
constexpr int kStateFloats = 4176;

struct NnWeightsF32 {
    const float *w0;          // [5][40][32]
    const float *dw_w[4];     // [kmax][cin] zero padded at the front for the shorter MixConv kernels
    const float *dw_b[4];     // [cin]
    const float *pw_w[4];     // [cin][64]   BatchNorm folded
    const float *pw_b[4];     // [64]
    const float *head_w;      // [17][64]
    const float *head_b;      // [1]
};

// input feature rows: a virtual sequence  pend[0..n_pend) ++ rows[0..n_rows)
struct NnInput {
    const float *ring0;       // [2][40] first-conv ring (rows -2, -1)
    const float *pend;        // [2][40] rows left over by the previous call
    int n_pend;
    const void *rows;         // [n_rows][40] uint16 (scaled by 1/25.6 on load) or float32
    int n_rows;
    int rows_are_f32;
};

MWW_HD float nn_virtual_row(const NnInput &in, int vr, int f) {
    // vr < 0: ring history; then pending rows; then this call's rows
    if (vr < 0) return in.ring0[(2 + vr) * kNumChannels + f];
    if (vr < in.n_pend) return in.pend[vr * kNumChannels + f];
    const int r = vr - in.n_pend;
    if (in.rows_are_f32) return static_cast<const float *>(in.rows)[(long long)r * kNumChannels + f];
    return (float)static_cast<const uint16_t *>(in.rows)[(long long)r * kNumChannels + f] * kFeatureScale;   // inference.py:93-94
}

// ---- phase: load ring state into the shared activation buffers (once per call) ----
template <int L>
MWW_HD void nn_load_state_l(int tid, float *sm, const float *state) {
    constexpr NnLayerGeom g = kGeom[L];
    const float *src = state + kStateOff[L + 1];
    // 4-byte cp.async (LDGSTS): the ~15 transposing copies a thread issues are all in flight at once instead of one
    // load -> store round trip after the other
    for (int e = tid; e < g.ring * g.cin; e += kNnThreads) {
        const int r = e / g.cin, c = e - r * g.cin;
        float *dst = sm + g.off + c * g.ld + (g.hp - g.ring) + r;
#if defined(__CUDA_ARCH__)
        asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((unsigned)__cvta_generic_to_shared(dst)), "l"(src + e));
#else
        *dst = src[e];
#endif
    }
}
MWW_HD void nn_load_state(int tid, float *sm, const float *state) {
    nn_load_state_l<0>(tid, sm, state); nn_load_state_l<1>(tid, sm, state); nn_load_state_l<2>(tid, sm, state);
    nn_load_state_l<3>(tid, sm, state); nn_load_state_l<4>(tid, sm, state);
}

// ---- phase: de-interleave the chunk's feature rows into three planes ----
// Chunk-relative row q = 0 .. 3n+1 is virtual row 3*step0 + q - 2 (q = 0, 1: the first-conv ring or the
// previous chunk's last two rows); plane[q % 3][f][q / 3].  Step t, tap j reads q = 3t + j.
MWW_HD void nn_load_features(int tid, float *sm, const NnInput &in, int step0, int n) {
    float *feat = sm + kXFloats + kDFloats;
    const int n_q = 3 * n + 2, U = n + 1;          // plane column u = q / 3 <= n
    // one thread handles 8 consecutive features of one row: a single 16-byte load on the uint16 fast path.
    // thread -> (8-feature group, plane j, u) with u FASTEST: consecutive lanes store consecutive words of a plane row
    // (row-major thread order puts the 32 lanes of a store on 2-3 banks).  The 16-byte global loads of neighbouring lanes are then 3 rows apart and meet in L1.
    for (int e = tid; e < 15 * U; e += kNnThreads) {
        const int u = e % U, jf = e / U, j = jf % 3, f0 = 8 * (jf / 3);
        const int q = 3 * u + j;
        if (q >= n_q) continue;
        const int vr = 3 * step0 + q - 2;
        float *dst = feat + (j * kNumChannels + f0) * kUS + u;
        const int r = vr - in.n_pend;
        if (vr >= in.n_pend && !in.rows_are_f32) {
            const uint16_t *src = static_cast<const uint16_t *>(in.rows) + (long long)r * kNumChannels + f0;
#if defined(__CUDA_ARCH__)
            const uint4 v = *reinterpret_cast<const uint4 *>(src);      // rows are 80 B apart, f0 * 2 is 16 B aligned
            const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                dst[(2 * i) * kUS] = (float)(w[i] & 0xFFFFu) * kFeatureScale;
                dst[(2 * i + 1) * kUS] = (float)(w[i] >> 16) * kFeatureScale;
            }
#else
            for (int i = 0; i < 8; ++i) dst[i * kUS] = (float)src[i] * kFeatureScale;
#endif
        } else {
#pragma unroll
            for (int i = 0; i < 8; ++i) dst[i * kUS] = nn_virtual_row(in, vr, f0 + i);
        }
    }
}

// ---- phase helper: stage block L's 1x1 weights [cin][64] into shared memory ----
// Two staging buffers alternate (even blocks: the feature-plane region, free once the first conv is done;
// odd blocks: a dedicated buffer) so block L+1's weights stream in (cp.async, no register round trip)
// while block L computes.
template <int L>
MWW_HD float *nn_pw_weight_buffer(float *sm) {
    return (L & 1) ? sm + kXFloats + kDFloats + kFeatFloats : sm + kXFloats + kDFloats;
}
template <int L>
MWW_HD void nn_stage_pw_weights(int tid, float *sm, const NnWeightsF32 &W) {
    float *wsm = nn_pw_weight_buffer<L>(sm);
    constexpr int n4 = kGeom[L].cin * 64 / 4;
    for (int e = tid; e < n4; e += kNnThreads) {
        const int k = e >> 4, c4 = e & 15;             // row k of [cin][64], 16-byte chunk c4
        float *dst = wsm + k * kWLdDev + 4 * c4;
#if defined(__CUDA_ARCH__)
        const unsigned d32 = (unsigned)__cvta_generic_to_shared(dst);
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d32), "l"(W.pw_w[L] + 4 * e));
#else
        for (int i = 0; i < 4; ++i) dst[i] = W.pw_w[L][4 * e + i];
#endif
    }
#if defined(__CUDA_ARCH__)
    asm volatile("cp.async.commit_group;" ::: "memory");
#endif
}
MWW_HD void nn_commit_group() {
#if defined(__CUDA_ARCH__)
    asm volatile("cp.async.commit_group;" ::: "memory");
#endif
}
// wait until at most N of this thread's cp.async groups are still in flight (no-op on the host)
template <int N>
MWW_HD void nn_wait_weights() {
#if defined(__CUDA_ARCH__)
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
#endif
}

// ---- phase: depthwise conv over (ring ++ chunk) for block L; output D[c][t] ----
// MixConv groups (mixednet.py:132-136): block 1 = 7 | 11 taps, block 2 = 9 | 15, blocks 0 and 3 uniform.  The
// container stores kernels zero padded at the front to kmax taps, so a K-tap group reads weights [kmax-K, kmax).
// cin = 64: 4 threads per channel x 9 steps (threads 256..287 idle); cin = 32: 9 threads per channel x 4 steps.
template <int L, int K, int TN>
MWW_HD void nn_depthwise_k(int c, int t0, float *sm, const NnWeightsF32 &W) {
    constexpr NnLayerGeom g = kGeom[L];
    float w[K];
#pragma unroll
    for (int j = 0; j < K; ++j) w[j] = W.dw_w[L][(g.kmax - K + j) * g.cin + c];
    const float bias = W.dw_b[L][c];
    float acc[TN];
#pragma unroll
    for (int i = 0; i < TN; ++i) acc[i] = 0.f;
    // output step t reads columns hp - (K-1) + t + j, j = 0..K-1 (oldest tap first, like the ring concat)
    const float *x = sm + g.off + c * g.ld + (g.hp - (K - 1)) + t0;
#pragma unroll
    for (int i = 0; i < TN + K - 1; ++i) {
        const float xv = x[i];
#pragma unroll
        for (int tt = 0; tt < TN; ++tt) {
            const int j = i - tt;
            if (j >= 0 && j < K) acc[tt] = fmaf(w[j], xv, acc[tt]);
        }
    }
    float *d = sm + kXFloats;
#pragma unroll
    for (int i = 0; i < TN; ++i) d[nn_d_index(c, t0 + i)] = acc[i] + bias;
}

template <int L>
MWW_HD void nn_depthwise(int tid, float *sm, const NnWeightsF32 &W) {
    constexpr NnLayerGeom g = kGeom[L];
    if (L == 0) {
        nn_depthwise_k<L, g.kmax, 4>(tid & 31, 4 * (tid >> 5), sm, W);
    } else {
        if (tid >= 256) return;
        const int c = tid & 63, t0 = 9 * (tid >> 6);
        if (L == 1) { if (c < 32) nn_depthwise_k<L, 7, 9>(c, t0, sm, W); else nn_depthwise_k<L, 11, 9>(c, t0, sm, W); }
        else if (L == 2) { if (c < 32) nn_depthwise_k<L, 9, 9>(c, t0, sm, W); else nn_depthwise_k<L, 15, 9>(c, t0, sm, W); }
        else nn_depthwise_k<L, g.kmax, 9>(c, t0, sm, W);
    }
}

// ---- phase: head, part 1: per-channel 17-tap partial sums into D[c][t] ----
MWW_HD void nn_head_partial(int tid, float *sm, const NnWeightsF32 &W) {
    constexpr NnLayerGeom g = kGeom[4];
    if (tid >= 256) return;
    const int c = tid & 63, t0 = 9 * (tid >> 6);
    float w[17];
#pragma unroll
    for (int j = 0; j < 17; ++j) w[j] = W.head_w[j * 64 + c];
    float acc[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) acc[i] = 0.f;
    const float *x = sm + g.off + c * g.ld + (g.hp - 16) + t0;
#pragma unroll
    for (int i = 0; i < 9 + 16; ++i) {
        const float xv = x[i];
#pragma unroll
        for (int tt = 0; tt < 9; ++tt) {
            const int j = i - tt;
            if (j >= 0 && j < 17) acc[tt] = fmaf(w[j], xv, acc[tt]);
        }
    }
    float *d = sm + kXFloats;
#pragma unroll
    for (int i = 0; i < 9; ++i) d[nn_d_index(c, t0 + i)] = acc[i];
}

MWW_HD float nn_sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }

// ---- phase: head, part 2: reduce over channels, bias, sigmoid ----
MWW_HD void nn_head_finish(int tid, float *sm, const NnWeightsF32 &W, int n, float *probs_out /* step0-relative */, float *logits_out) {
    if (tid >= kTT || tid >= n) return;
    const float *d = sm + kXFloats;
    float acc = 0.f;
    for (int c = 0; c < 64; ++c) acc += d[nn_d_index(c, tid)];
    const float logit = acc + W.head_b[0];
    if (logits_out) logits_out[tid] = logit;
    probs_out[tid] = nn_sigmoid(logit);
}

// ---- phase pair: slide the ring histories left by n steps (read -> barrier -> write) ----
constexpr int kShiftPerThread = 5;   // ceil(64*22 / 288)
template <int L>
MWW_HD void nn_shift_read_l(int tid, const float *sm, int n, float (&tmp)[kShiftPerThread]) {
    constexpr NnLayerGeom g = kGeom[L];
#pragma unroll
    for (int q = 0; q < kShiftPerThread; ++q) {
        const int e = tid + q * kNnThreads;
        if (e < g.ring * g.cin) {
            const int c = e / g.ring, r = e - c * g.ring;
            tmp[q] = sm[g.off + c * g.ld + (g.hp - g.ring) + n + r];
        }
    }
}
template <int L>
MWW_HD void nn_shift_write_l(int tid, float *sm, const float (&tmp)[kShiftPerThread]) {
    constexpr NnLayerGeom g = kGeom[L];
#pragma unroll
    for (int q = 0; q < kShiftPerThread; ++q) {
        const int e = tid + q * kNnThreads;
        if (e < g.ring * g.cin) {
            const int c = e / g.ring, r = e - c * g.ring;
            sm[g.off + c * g.ld + (g.hp - g.ring) + r] = tmp[q];
        }
    }
}
MWW_HD void nn_shift_read(int tid, const float *sm, int n, float (&tmp)[5][kShiftPerThread]) {
    nn_shift_read_l<0>(tid, sm, n, tmp[0]); nn_shift_read_l<1>(tid, sm, n, tmp[1]); nn_shift_read_l<2>(tid, sm, n, tmp[2]);
    nn_shift_read_l<3>(tid, sm, n, tmp[3]); nn_shift_read_l<4>(tid, sm, n, tmp[4]);
}
MWW_HD void nn_shift_write(int tid, float *sm, const float (&tmp)[5][kShiftPerThread]) {
    nn_shift_write_l<0>(tid, sm, tmp[0]); nn_shift_write_l<1>(tid, sm, tmp[1]); nn_shift_write_l<2>(tid, sm, tmp[2]);
    nn_shift_write_l<3>(tid, sm, tmp[3]); nn_shift_write_l<4>(tid, sm, tmp[4]);
}

// ---- phases: write the ring state, first-conv ring and pending rows back (once per call) ----
template <int L>
MWW_HD void nn_store_state_l(int tid, const float *sm, float *state) {
    constexpr NnLayerGeom g = kGeom[L];
    float *dst = state + kStateOff[L + 1];
    for (int e = tid; e < g.ring * g.cin; e += kNnThreads) {
        const int r = e / g.cin, c = e - r * g.cin;
        dst[e] = sm[g.off + c * g.ld + (g.hp - g.ring) + r];
    }
}
// The new first-conv ring (two rows preceding the next unconsumed row) and the new pending rows are
// gathered from the OLD ring/pending/rows first; a barrier separates this from nn_tail_write.
struct NnTail { float ring_new, pend_new; };
MWW_HD void nn_tail_read(int tid, const NnInput &in, int n_steps, int n_virtual_rows, NnTail &t) {
    const int consumed = 3 * n_steps;
    t.ring_new = 0.f; t.pend_new = 0.f;
    if (tid < 2 * kNumChannels) {
        const int r = tid / kNumChannels, f = tid - r * kNumChannels;
        t.ring_new = nn_virtual_row(in, consumed - 2 + r, f);
        const int vr = consumed + r;
        t.pend_new = vr < n_virtual_rows ? nn_virtual_row(in, vr, f) : 0.f;
    }
}
MWW_HD void nn_tail_write(int tid, const float *sm, float *state, float *pend_out, const NnTail &t) {
    nn_store_state_l<0>(tid, sm, state); nn_store_state_l<1>(tid, sm, state); nn_store_state_l<2>(tid, sm, state);
    nn_store_state_l<3>(tid, sm, state); nn_store_state_l<4>(tid, sm, state);
    if (tid < 2 * kNumChannels) { state[tid] = t.ring_new; pend_out[tid] = t.pend_new; }
}

}  // namespace mww
