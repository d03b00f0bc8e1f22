// mww_nn_live.cuh -- fp32 MixedNet, LIVE-STEP formulation: one model step (three new 10 ms feature rows) for
// many streams per launch -- the literal shape of the reference's hot loop (set_tensor / invoke / get_tensor once
// per 30 ms, microwakeword/inference.py:109-123), batched over streams instead of repeated per stream.
//
// The clip kernels (mww_nn_dev.cuh) amortise the ring state over many steps of one stream; with one step per call
// there is nothing to amortise, the ring state (4 176 floats per stream, stream.py:581-595) has to cross HBM once
// per step and the kernel is HBM-bound (SURVEY.md 8d "live step": ~18.8 KB per stream-step algorithmic).  So here a
// CTA owns 32 STREAMS: the stream index is the M dimension of the tensor-core contractions (first conv, 1x1
// projections: same 3xTF32 mma path as the clip kernel), all 1x1 weights stay resident in shared memory, and the
// depthwise / head stages stream each (stream, channel) ring column through registers: load R rows (coalesced
// over channels), accumulate the taps, and write ONLY the new row over the oldest one: between live calls every ring is
// kept ROTATED (LiveHeads: the physical row that holds the oldest logical row; all streams of a handle advance in
// lockstep so one head per ring serves every stream), which is the concat(state, input)[-R:] update of
// stream.py:584-590 without moving R - 1 rows through HBM.  Per stream-step that is the SURVEY.md 8d algorithmic
// traffic: the ring read once (16.7 KB) + one new row per ring written (1.5 KB), not 2 x 16.7 KB.
// Rings are rotated back to the canonical (oldest-first) layout of the clip kernels by live_canonicalise_column
// whenever a clip call, mww_get_state or a mode switch needs it, so clip and live calls can still be mixed.
#pragma once

#include "mww_nn_mma.cuh"

namespace mww {

// physical row of the oldest logical row of each rotating ring: MixConv blocks 0..3, then the head ring
struct LiveHeads { int h[5]; };
constexpr int kLiveRingRows[5] = {4, 10, 14, 22, 16};      // host-side copy (device code uses the functions below)
MWW_HD constexpr int live_ring_rows(int i) { return i == 0 ? 4 : (i == 1 ? 10 : (i == 2 ? 14 : (i == 3 ? 22 : 16))); }
MWW_HD constexpr int live_ring_cols(int i) { return i == 0 ? 32 : 64; }

constexpr int kLiveThreads = 256;
constexpr int kLiveStreams = 32;                  // streams per CTA = two 16-row MMA tiles
constexpr int kLivePitch = 40;                    // [k][stream] pitch: 40 = 8 (mod 32) -> conflict-free A fragments
// shared memory (floats): 1x1 weights of the four blocks (pitch kWLd), A operand of the first conv [200][40],
// H = new activation row of every stream [64][40], D = depthwise output [64][40]
constexpr int kLiveOffPw0 = 0;                    // block 0's 32x64 weights are NOT staged (read from L2): keeps 2 CTAs / SM
constexpr int kLiveOffPw1 = 0;
constexpr int kLiveOffPw2 = kLiveOffPw1 + 64 * kWLd;
constexpr int kLiveOffPw3 = kLiveOffPw2 + 64 * kWLd;
constexpr int kLiveOffA = kLiveOffPw3 + 64 * kWLd;
constexpr int kLiveOffH = kLiveOffA + 200 * kLivePitch;
constexpr int kLiveOffD = kLiveOffH + 64 * kLivePitch;
constexpr int kLiveSmemFloats = kLiveOffD + 64 * kLivePitch;
constexpr int kLiveSmemBytes = kLiveSmemFloats * 4;           // 107.8 KB -> 2 CTAs / SM (16 warps), persistent over stream groups

template <int L>
MWW_HD int live_pw_offset() { return L == 0 ? kLiveOffPw0 : (L == 1 ? kLiveOffPw1 : (L == 2 ? kLiveOffPw2 : kLiveOffPw3)); }

// ---- once per CTA: stage all 1x1 weights ----
MWW_HD void live_load_weights(int tid, float *sm, const NnWeightsF32 &W) {
    for (int L = 1; L < 4; ++L) {
        float *dst = sm + (L == 1 ? kLiveOffPw1 : (L == 2 ? kLiveOffPw2 : kLiveOffPw3));
        for (int e = tid; e < 64 * 64; e += kLiveThreads) dst[(e >> 6) * kWLd + (e & 63)] = W.pw_w[L][e];
    }
}

// virtual feature row vr of one stream: pending rows first, then the three new rows (this call's input)
struct LiveInput {
    const float *state;        // [S][4176]
    const float *pend;         // [S][2][40]
    int n_pend;
    const void *rows;          // [S][3][40] uint16 or float32
    long long rows_stream_stride_bytes;
    int rows_are_f32;
};
// One stream's first-conv window is a plain concatenation of three contiguous arrays:
//     window[0:200] = state[0:80] (the 2-row first-conv ring) ++ pend[0:40 p] ++ rows[0:40 (3 - p)],     p = n_pend
// and the call leaves   new ring = window[120:200]   and   new pend = rows[40 (3 - p) : 120]  (p rows).
// All indices are kept NON-NEGATIVE and unsigned on purpose: with a signed "virtual row - 2" formulation nvcc 12.9
// re-associated (2 + vr) * 40 into a negative 32-bit term that was then added to the 64-bit address without sign
// extension (a 16 GB stray access, caught by compute-sanitizer).
MWW_HD float live_row_value(const LiveInput &in, size_t su, unsigned e) {
    const char *base = static_cast<const char *>(in.rows) + su * (size_t)in.rows_stream_stride_bytes;
    if (in.rows_are_f32) return reinterpret_cast<const float *>(base)[e];
    return (float)reinterpret_cast<const uint16_t *>(base)[e] * kFeatureScale;
}

// ---- phase: A[k = tap*40 + f][stream] for the first conv.  A warp owns 4 of the group's 32 streams; lane l reads
// window elements l, l + 32, ... (coalesced, 7 independent loads per stream) and keeps them: after the barrier the
// holders of window[120:200] write the new first-conv ring, and 3 more values per lane become the new pending rows.
constexpr int kLiveKeep = 10;         // per thread and stream: 7 window values + 3 new-pending values
// Every load below is UNCONDITIONAL on a clamped, always-valid address and the value is selected afterwards: with
// conditional loads the compiler emitted one branch per element and the 40 loads of a thread serialised into 40
// dependent DRAM round trips.
template <bool F32ROWS>
MWW_HD void live_build_a_t(int tid, float *sm, const LiveInput &in, long long s0, int n_valid, float (&keep)[4][kLiveKeep]) {
    const int warp = tid >> 5;
    const unsigned lane = (unsigned)(tid & 31), np40 = (unsigned)in.n_pend * (unsigned)kNumChannels;
    float *a = sm + kLiveOffA;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const int sl = warp * 4 + q;
        const bool ok = sl < n_valid;
        const size_t su = (size_t)(s0 + (ok ? sl : 0));
        const float *st = in.state + su * (size_t)kStateFloats;
        const float *pd = in.pend + su * (size_t)(2 * kNumChannels);
        const char *rb = static_cast<const char *>(in.rows) + su * (size_t)in.rows_stream_stride_bytes;
        const float *rf = reinterpret_cast<const float *>(rb);
        const uint16_t *r16 = reinterpret_cast<const uint16_t *>(rb);
#pragma unroll
        for (int i = 0; i < 7; ++i) {
            const unsigned k = lane + 32u * (unsigned)i, kk = k < 199u ? k : 199u;
            const bool in_ring = kk < 80u, in_pend = !in_ring && kk < 80u + np40, is_row = !in_ring && !in_pend;
            const unsigned e = is_row ? kk - 80u - np40 : 0u;
            const float *fp = in_ring ? st + kk : (in_pend ? pd + (kk - 80u) : (F32ROWS ? rf + e : st));
            float v = *fp;
            if (!F32ROWS) {
                const float u = (float)r16[e] * kFeatureScale;
                v = is_row ? u : v;
            }
            v = (ok && k < 200u) ? v : 0.f;
            keep[q][i] = v;
            if (k < 200u) a[k * (unsigned)kLivePitch + (unsigned)sl] = v;
        }
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            const unsigned e2 = lane + 32u * (unsigned)i;
            const bool live = ok && e2 < np40;
            const unsigned idx = live ? 3u * (unsigned)kNumChannels - np40 + e2 : 0u;
            const float v = F32ROWS ? rf[idx] : (float)r16[idx] * kFeatureScale;
            keep[q][7 + i] = live ? v : 0.f;
        }
    }
}
MWW_HD void live_build_a(int tid, float *sm, const LiveInput &in, long long s0, int n_valid, float (&keep)[4][kLiveKeep]) {
    if (in.rows_are_f32) live_build_a_t<true>(tid, sm, in, s0, n_valid, keep);
    else live_build_a_t<false>(tid, sm, in, s0, n_valid, keep);
}
// after a barrier (every read of the old ring / pending rows is done): new ring = window[120:200], new pending rows
MWW_HD void live_write_tail(int tid, float *state, float *pend, long long s0, int n_valid, const float (&keep)[4][kLiveKeep]) {
    const int warp = tid >> 5;
    const unsigned lane = (unsigned)(tid & 31);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const int sl = warp * 4 + q;
        if (sl >= n_valid) continue;
        const size_t su = (size_t)(s0 + sl);
#pragma unroll
        for (int i = 3; i < 7; ++i) {
            const unsigned k = lane + 32u * (unsigned)i;
            if (k >= 120u && k < 200u) state[su * (size_t)kStateFloats + (k - 120u)] = keep[q][i];
        }
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            const unsigned e = lane + 32u * (unsigned)i;
            if (e < 80u) pend[su * (size_t)(2 * kNumChannels) + e] = keep[q][7 + i];
        }
    }
}

// ---- first conv epilogue: ReLU into H[o][stream] ----
MWW_HD void live_fc_store_tile(float *sm, int r0, int n0, int lane, const float (&c)[4]) {
    const int g = lane >> 2, tig = lane & 3;
    float *h = sm + kLiveOffH;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int row = r0 + g + ((i & 2) ? 8 : 0), o = n0 + 2 * tig + (i & 1);
        h[o * kLivePitch + row] = c[i] > 0.f ? c[i] : 0.f;
    }
}
// `bias` = the block's 64 folded-BatchNorm biases (global memory in v1, shared memory in v2)
MWW_HD void live_pw_store_tile_b(float *sm, const float *bias, int r0, int n0, int lane, const float (&c)[4]) {
    const int g = lane >> 2, tig = lane & 3;
    float *h = sm + kLiveOffH;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int row = r0 + g + ((i & 2) ? 8 : 0), o = n0 + 2 * tig + (i & 1);
        const float v = c[i] + bias[o];
        h[o * kLivePitch + row] = v > 0.f ? v : 0.f;
    }
}
template <int L>
MWW_HD void live_pw_store_tile(float *sm, const NnWeightsF32 &W, int r0, int n0, int lane, const float (&c)[4]) {
    live_pw_store_tile_b(sm, W.pw_b[L], r0, n0, lane, c);
}

// ---- depthwise of block L for (stream, channel) columns: ring rows stream through registers ----
// thread -> channel c = tid % cin, stream subgroup = tid / cin; each thread walks kLiveStreams * cin / 256 streams,
// U at a time: the kernel is bound by HBM latency (one 8-warp CTA per SM), so U ring columns (U * R independent
// loads) are put in flight before any of them is consumed.
// w[p] must already be the tap of PHYSICAL row p (i.e. of logical row (p - head) mod R); w[R] is the new row's tap.
template <int R, int CIN, int U>
MWW_HD void live_ring_pass(float *const (&ring)[U], const bool (&ok)[U], const float (&w)[R + 1], const float (&xn)[U], float bias, int head,
                           float (&out)[U]) {
    float x[U][R];
#pragma unroll
    for (int u = 0; u < U; ++u)
#pragma unroll
        for (int r = 0; r < R; ++r) x[u][r] = ok[u] ? ring[u][r * CIN] : 0.f;
#pragma unroll
    for (int u = 0; u < U; ++u) {
        float acc = bias;
#pragma unroll
        for (int r = 0; r < R; ++r) acc = fmaf(w[r], x[u][r], acc);
        out[u] = fmaf(w[R], xn[u], acc);
        if (ok[u]) ring[u][head * CIN] = xn[u];          // overwrite the oldest row; the caller advances the head
    }
}

template <int L>
MWW_HD void live_depthwise(int tid, float *sm, const NnWeightsF32 &W, float *state, long long s0, int n_valid, int head) {
    constexpr NnLayerGeom g = kGeom[L];
    constexpr int R = g.ring;
    constexpr int per = kLiveStreams * g.cin / kLiveThreads;     // streams per thread: 4 (cin 32) or 8 (cin 64)
    constexpr int U = L == 3 ? 2 : 4;
    constexpr int ring_off = kStateOff[L + 1];
    const int c = tid % g.cin, sub = tid / g.cin;
    float w[R + 1];
#pragma unroll
    for (int p = 0; p <= R; ++p) {                                        // kmax = R + 1; zero padded at the front for short MixConv kernels
        const int j = p == R ? R : (p - head < 0 ? p - head + R : p - head);
        w[p] = W.dw_w[L][j * g.cin + c];
    }
    const float bias = W.dw_b[L][c];
    const float *h = sm + kLiveOffH + c * kLivePitch;
    float *d = sm + kLiveOffD + c * kLivePitch;
#pragma unroll 1
    for (int i = 0; i < per; i += U) {
        float *ring[U]; bool ok[U]; float xn[U], out[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int sl = sub * per + i + u;
            ok[u] = sl < n_valid;
            ring[u] = state + (size_t)(s0 + (ok[u] ? sl : 0)) * kStateFloats + ring_off + c;
            xn[u] = h[sl];
        }
        live_ring_pass<R, g.cin, U>(ring, ok, w, xn, bias, head, out);
#pragma unroll
        for (int u = 0; u < U; ++u) d[sub * per + i + u] = ok[u] ? out[u] : 0.f;
    }
}

// ---- head: 17-tap dot per (stream, channel) into D, ring shifted; then reduce over channels ----
MWW_HD void live_head_partial(int tid, float *sm, const NnWeightsF32 &W, float *state, long long s0, int n_valid, int head) {
    constexpr int per = kLiveStreams * 64 / kLiveThreads;        // 8
    constexpr int U = 4;
    constexpr int ring_off = kStateOff[5];
    const int c = tid & 63, sub = tid >> 6;
    float w[17];
#pragma unroll
    for (int p = 0; p < 17; ++p) {
        const int j = p == 16 ? 16 : (p - head < 0 ? p - head + 16 : p - head);
        w[p] = W.head_w[j * 64 + c];
    }
    const float *h = sm + kLiveOffH + c * kLivePitch;
    float *d = sm + kLiveOffD + c * kLivePitch;
#pragma unroll 1
    for (int i = 0; i < per; i += U) {
        float *ring[U]; bool ok[U]; float xn[U], out[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int sl = sub * per + i + u;
            ok[u] = sl < n_valid;
            ring[u] = state + (size_t)(s0 + (ok[u] ? sl : 0)) * kStateFloats + ring_off + c;
            xn[u] = h[sl];
        }
        live_ring_pass<16, 64, U>(ring, ok, w, xn, 0.f, head, out);
#pragma unroll
        for (int u = 0; u < U; ++u) d[sub * per + i + u] = ok[u] ? out[u] : 0.f;
    }
}
MWW_HD void live_head_finish_b(int tid, const float *sm, float head_bias, long long s0, int n_valid, float *probs, long long probs_stride) {
    if (tid >= kLiveStreams || tid >= n_valid) return;
    const float *d = sm + kLiveOffD + tid;
    float acc = 0.f;
    for (int c = 0; c < 64; ++c) acc += d[c * kLivePitch];
    probs[(s0 + tid) * probs_stride] = nn_sigmoid(acc + head_bias);
}
MWW_HD void live_head_finish(int tid, const float *sm, const NnWeightsF32 &W, long long s0, int n_valid, float *probs, long long probs_stride) {
    live_head_finish_b(tid, sm, W.head_b[0], s0, n_valid, probs, probs_stride);
}

// ---- back to the canonical layout: one (stream, ring, channel) column per call ----
// col in [0, 288): ring i owns kLiveRingCols[i] consecutive columns.
MWW_HD void live_canonicalise_column(float *state, long long s, int col, const LiveHeads &heads) {
    int i = 0, c = col;
    while (c >= live_ring_cols(i)) { c -= live_ring_cols(i); ++i; }
    const int R = live_ring_rows(i), C = live_ring_cols(i), h = heads.h[i];
    if (h == 0) return;
    int off = 2 * kNumChannels;
    for (int k = 0; k < i; ++k) off += live_ring_rows(k) * live_ring_cols(k);
    float *ring = state + (size_t)s * kStateFloats + off + c;
    float tmp[22];
    for (int j = 0; j < R; ++j) { const int p = h + j >= R ? h + j - R : h + j; tmp[j] = ring[p * C]; }
    for (int j = 0; j < R; ++j) ring[j * C] = tmp[j];
}

// =====================================================================================================================
// v2: warp-specialised live step.  The kernel above runs latency-bound: a CTA's ring loads and its layer chain take
// turns.  The old ring rows do not depend on this step's activations, so
//     P[column] = bias + sum over the R old rows of tap(row) * x(row)           ("streamers", 16 warps)
// can be computed for stream group g+1 while the layer chain of group g runs   ("chain", 8 warps)
//     first conv -> { D = fma(tap_new, x_new, P) ; store x_new over the oldest ring row ; 1x1 + ReLU } x 4 -> head.
// The arithmetic and its order are exactly those of live_ring_pass, so the two kernels are bit-identical.  One CTA of 768
// threads per SM, P double-buffered in shared memory and handed over with named barriers; the streamers keep R (or 2 R)
// independent 128-byte row segments in flight per thread all the time, which is what an HBM-bound kernel wants.
constexpr int kLive2ChainThreads = 256;
constexpr int kLive2StreamThreads = 512;
constexpr int kLive2Threads = kLive2ChainThreads + kLive2StreamThreads;
constexpr int kLive2PPitch = 33;                              // P[column][stream]: odd pitch -> conflict-free on both sides
constexpr int kLive2Cols = 32 + 64 * 4;                       // 288 ring columns per stream (blocks 0..3, head)
constexpr int kLive2PFloats = kLive2Cols * kLive2PPitch;      // one P buffer
constexpr int kLive2OffP = kLiveSmemFloats;                   // the chain's regions keep their v1 offsets
// Everything the CHAIN reads besides its own activations lives in shared memory: with the first conv's and block 0's weights,
// the newest taps and the biases coming from L2 / L1, every dependent global access of the latency-bound chain waits behind the
// streamers, which keep the memory system saturated.  (The streamers' old-row taps moved the other way, to L1-cached global reads, to make room.)
constexpr int kLive2W0Pitch = 40;                             // first-conv weights [200][40]: pitch = 8 (mod 32) like kWLd
constexpr int kLive2OffPw0 = kLive2OffP + 2 * kLive2PFloats;
constexpr int kLive2OffSmall = kLive2OffPw0 + 32 * kWLd;      // newest taps [288], depthwise... 1x1 biases [4][64], head bias
constexpr int kLive2SmallTaps = 0, kLive2SmallPwBias = kLive2Cols, kLive2SmallHeadBias = kLive2Cols + 256;
constexpr int kLive2OffW0 = kLive2OffSmall + kLive2Cols + 256 + 32;   // last: v3 puts its bulk-copy stages here instead (128-byte aligned)
constexpr int kLive2SmemFloats = kLive2OffW0 + 200 * kLive2W0Pitch;
constexpr int kLive2SmemBytes = kLive2SmemFloats * 4;         // 227.3 KB of the 227 KB (232 448 B) a CTA may have
static_assert((kLive2OffW0 * 4) % 128 == 0, "stage alignment");
static_assert(kLive2SmemBytes <= 232448, "shared memory per CTA");
MWW_HD constexpr int live2_col_base(int i) { return i == 0 ? 0 : 32 + 64 * (i - 1); }
MWW_HD constexpr int live2_wrot_base(int i) { return i == 0 ? 0 : (i == 1 ? 128 : (i == 2 ? 128 + 640 : (i == 3 ? 128 + 640 + 896 : 128 + 640 + 896 + 1408))); }

// once per CTA: the chain's constants
MWW_HD void live2_stage_chain_tables(int tid, int n_threads, float *sm, const NnWeightsF32 &W, bool with_w0 = true) {
    if (with_w0)
        for (int e = tid; e < 200 * 32; e += n_threads) sm[kLive2OffW0 + (e >> 5) * kLive2W0Pitch + (e & 31)] = W.w0[e];
    for (int e = tid; e < 32 * 64; e += n_threads) sm[kLive2OffPw0 + (e >> 6) * kWLd + (e & 63)] = W.pw_w[0][e];
    float *small = sm + kLive2OffSmall;
    for (int e = tid; e < kLive2Cols; e += n_threads) {        // newest tap (row R of the [R + 1][C] table) of every ring column
        int i = 0, c = e;
        while (c >= live_ring_cols(i)) { c -= live_ring_cols(i); ++i; }
        small[kLive2SmallTaps + e] = (i < 4 ? W.dw_w[i] : W.head_w)[live_ring_rows(i) * live_ring_cols(i) + c];
    }
    for (int e = tid; e < 256; e += n_threads) small[kLive2SmallPwBias + e] = W.pw_b[e >> 6][e & 63];
    if (tid == 0) small[kLive2SmallHeadBias] = W.head_b[0];
}

// Streamer thread <-> (stream, FOUR consecutive channels): C / 4 neighbouring lanes read one whole ring row with 16-byte
// loads, so a ring costs a quarter of the load instructions / L1 requests of the one-channel-per-thread mapping (the chain's
// shared-memory traffic goes through the same LSU pipe).  Rows are taken CH at a time and double-buffered: the loads of chunk
// k + 1 are issued before the multiply-adds of chunk k.  Multiply-adds run in physical row order (bit-identical sums); the
// tap of physical row r is row (r - head) mod R of the [R + 1][C] table, read through L1 as one 16-byte load per row.
struct Quad { float x, y, z, w; };
MWW_HD Quad load_quad(const float *p) {
#if defined(__CUDA_ARCH__)
    const float4 v = *reinterpret_cast<const float4 *>(p);
    return Quad{v.x, v.y, v.z, v.w};
#else
    return Quad{p[0], p[1], p[2], p[3]};
#endif
}
MWW_HD Quad load_quad_ro(const float *p) {
#if defined(__CUDA_ARCH__)
    const float4 v = __ldg(reinterpret_cast<const float4 *>(p));
    return Quad{v.x, v.y, v.z, v.w};
#else
    return Quad{p[0], p[1], p[2], p[3]};
#endif
}
template <int I>
MWW_HD void live2_stream_ring(int st, const NnWeightsF32 &W, const float *state, long long s0, int n_valid, int head, float *p_buf) {
    constexpr int R = live_ring_rows(I), C = live_ring_cols(I);
    constexpr int lanes = C / 4;                                       // threads per stream: 8 (block 0) or 16
    constexpr int CH = R == 4 ? 4 : (R == 10 ? 5 : (R == 14 ? 7 : (R == 22 ? 11 : 8)));   // rows per chunk
    constexpr int NCH = R / CH;
    static_assert(R % CH == 0, "row chunking");
    constexpr int ring_off = kStateOff[I + 1];
    const int sl = st / lanes, c = 4 * (st % lanes);
    if (sl >= kLiveStreams) return;                                    // block 0 needs only half of the streamer threads
    const bool ok = sl < n_valid;
    const float *ring = state + (size_t)(s0 + (ok ? sl : 0)) * kStateFloats + ring_off + c;
    const float *taps = (I < 4 ? W.dw_w[I < 4 ? I : 0] : W.head_w) + c;
    const int j0 = head == 0 ? 0 : R - head;
    Quad acc;
    if (I < 4) acc = load_quad_ro(W.dw_b[I < 4 ? I : 0] + c); else acc = Quad{0.f, 0.f, 0.f, 0.f};
    Quad x[2][CH];
#pragma unroll
    for (int r = 0; r < CH; ++r) x[0][r] = ok ? load_quad(ring + r * C) : Quad{0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < NCH; ++k) {
        if (k + 1 < NCH) {
#pragma unroll
            for (int r = 0; r < CH; ++r) x[(k + 1) & 1][r] = ok ? load_quad(ring + ((k + 1) * CH + r) * C) : Quad{0.f, 0.f, 0.f, 0.f};
        }
#pragma unroll
        for (int r = 0; r < CH; ++r) {
            const int pr = k * CH + r;
            const int j = pr < head ? j0 + pr : pr - head;                 // (pr - head) mod R
            const Quad w = load_quad_ro(taps + j * C);
            const Quad v = x[k & 1][r];
            acc.x = fmaf(w.x, v.x, acc.x); acc.y = fmaf(w.y, v.y, acc.y);
            acc.z = fmaf(w.z, v.z, acc.z); acc.w = fmaf(w.w, v.w, acc.w);
        }
    }
    float *p_col = p_buf + (live2_col_base(I) + c) * kLive2PPitch + sl;
    p_col[0] = acc.x; p_col[kLive2PPitch] = acc.y; p_col[2 * kLive2PPitch] = acc.z; p_col[3 * kLive2PPitch] = acc.w;
}
MWW_HD void live2_stream_group(int st, const NnWeightsF32 &W, const float *state, long long s0, int n_valid, const LiveHeads &heads, float *p_buf) {
    live2_stream_ring<3>(st, W, state, s0, n_valid, heads.h[3], p_buf);        // longest rings first: their loads overlap the rest
    live2_stream_ring<4>(st, W, state, s0, n_valid, heads.h[4], p_buf);
    live2_stream_ring<2>(st, W, state, s0, n_valid, heads.h[2], p_buf);
    live2_stream_ring<1>(st, W, state, s0, n_valid, heads.h[1], p_buf);
    live2_stream_ring<0>(st, W, state, s0, n_valid, heads.h[0], p_buf);
}

// chain: first-conv window without per-thread copies kept across the barrier (the new first-conv ring is read back from
// the A operand, the new pending rows from the caller's rows)
// NT = threads that share the work (512: the streamers build the window one group ahead of the chain; a chain loading it
// itself stalls here, its loads queue behind the streamers' in the LSU)
template <bool F32ROWS, int NT>
MWW_HD void live2_build_a_t(int tid, float *sm, const LiveInput &in, long long s0, int n_valid) {
    constexpr int QPW = kLiveStreams / (NT / 32);                  // streams per warp
    const int warp = tid >> 5;
    const unsigned lane = (unsigned)(tid & 31), np40 = (unsigned)in.n_pend * (unsigned)kNumChannels;
    float *a = sm + kLiveOffA;
#pragma unroll
    for (int q = 0; q < QPW; ++q) {
        const int sl = warp * QPW + q;
        const bool ok = sl < n_valid;
        const size_t su = (size_t)(s0 + (ok ? sl : 0));
        const float *st = in.state + su * (size_t)kStateFloats;
        const float *pd = in.pend + su * (size_t)(2 * kNumChannels);
        const char *rb = static_cast<const char *>(in.rows) + su * (size_t)in.rows_stream_stride_bytes;
        const float *rf = reinterpret_cast<const float *>(rb);
        const uint16_t *r16 = reinterpret_cast<const uint16_t *>(rb);
#pragma unroll
        for (int i = 0; i < 7; ++i) {
            const unsigned k = lane + 32u * (unsigned)i, kk = k < 199u ? k : 199u;
            const bool in_ring = kk < 80u, in_pend = !in_ring && kk < 80u + np40, is_row = !in_ring && !in_pend;
            const unsigned e = is_row ? kk - 80u - np40 : 0u;
            const float *fp = in_ring ? st + kk : (in_pend ? pd + (kk - 80u) : (F32ROWS ? rf + e : st));
            float v = *fp;
            if (!F32ROWS) {
                const float u = (float)r16[e] * kFeatureScale;
                v = is_row ? u : v;
            }
            v = (ok && k < 200u) ? v : 0.f;
            if (k < 200u) a[k * (unsigned)kLivePitch + (unsigned)sl] = v;
        }
    }
}
template <int NT>
MWW_HD void live2_build_a(int tid, float *sm, const LiveInput &in, long long s0, int n_valid) {
    if (in.rows_are_f32) live2_build_a_t<true, NT>(tid, sm, in, s0, n_valid);
    else live2_build_a_t<false, NT>(tid, sm, in, s0, n_valid);
}
// v3: the same window in two halves -- the loads of group k + 1 are issued (into registers) right after group k's window went
// to shared memory, i.e. a whole chain period before they are needed: under the bulk copies' HBM load a round of global
// loads costs microseconds, and A is free only after the first conv of the previous group (window warps loading on demand
// leave the chain waiting for A).  The same warps also move the call's last n_pend
// rows into the pending-row buffer (v1 / v2: the chain does, with loads on its critical path): a stream's old pending rows
// are read (they are part of the window) before its new ones are written (a named barrier among the window warps).
// 192 threads: thread t owns the (stream, element) pairs t, t + 192, ... of the group's 32 x 200 -- 34 values per thread, no
// spills at the kernel's 80 registers (128 threads x 56 values spill).
constexpr int kLive3WindowThreads = 192;
constexpr int kLive3WindowPerThread = (kLiveStreams * 200 + kLive3WindowThreads - 1) / kLive3WindowThreads;     // 34
template <bool F32ROWS>
MWW_HD void live3_window_load_t(int t, const LiveInput &in, long long s0, int n_valid, float (&v)[kLive3WindowPerThread]) {
    const unsigned np40 = (unsigned)in.n_pend * (unsigned)kNumChannels;
#pragma unroll
    for (int i = 0; i < kLive3WindowPerThread; ++i) {
        const unsigned idx = (unsigned)t + (unsigned)(kLive3WindowThreads * i), slr = idx / 200u, sl = slr < 31u ? slr : 31u, kk = idx - 200u * slr;
        const bool ok = (int)sl < n_valid && idx < (unsigned)(kLiveStreams * 200);
        const size_t su = (size_t)(s0 + (ok ? (int)sl : 0));
        const float *st = in.state + su * (size_t)kStateFloats;
        const float *pd = in.pend + su * (size_t)(2 * kNumChannels);
        const char *rb = static_cast<const char *>(in.rows) + su * (size_t)in.rows_stream_stride_bytes;
        const bool in_ring = kk < 80u, in_pend = !in_ring && kk < 80u + np40, is_row = !in_ring && !in_pend && kk < 200u;
        const unsigned e = is_row ? kk - 80u - np40 : 0u;
        const float *fp = in_ring ? st + kk : (in_pend ? pd + (kk - 80u) : (F32ROWS ? reinterpret_cast<const float *>(rb) + e : st));
        float x = *fp;
        if (!F32ROWS) {
            const float u = (float)reinterpret_cast<const uint16_t *>(rb)[e] * kFeatureScale;
            x = is_row ? u : x;
        }
        v[i] = ok ? x : 0.f;
    }
}
MWW_HD void live3_window_load(int t, const LiveInput &in, long long s0, int n_valid, float (&v)[kLive3WindowPerThread]) {
    if (in.rows_are_f32) live3_window_load_t<true>(t, in, s0, n_valid, v);
    else live3_window_load_t<false>(t, in, s0, n_valid, v);
}
// the call's last n_pend rows -> pending-row buffer (after every window thread has read the old pending rows: caller's barrier)
MWW_HD void live3_pend_store(int t, const LiveInput &in, float *pend_out, long long s0, int n_valid) {
    const unsigned np40 = (unsigned)in.n_pend * (unsigned)kNumChannels;
    for (unsigned idx = (unsigned)t; idx < (unsigned)n_valid * np40; idx += (unsigned)kLive3WindowThreads) {
        const unsigned sl = idx / np40, e = idx - sl * np40;
        const size_t su = (size_t)(s0 + sl);
        pend_out[su * (size_t)(2 * kNumChannels) + e] = live_row_value(in, su, (unsigned)(3 * kNumChannels) - np40 + e);
    }
}
MWW_HD void live3_window_store(int t, float *sm, const float (&v)[kLive3WindowPerThread]) {
    float *a = sm + kLiveOffA;
#pragma unroll
    for (int i = 0; i < kLive3WindowPerThread; ++i) {
        const unsigned idx = (unsigned)t + (unsigned)(kLive3WindowThreads * i), sl = idx / 200u, kk = idx - 200u * sl;
        if (idx < (unsigned)(kLiveStreams * 200)) a[kk * (unsigned)kLivePitch + sl] = v[i];
    }
}
// v3 "P" thread: ring I, column c of it.  Taps rotated once per launch so that tap r multiplies PHYSICAL row r of the rotated
// ring (tap of physical row r = row (r - head) mod R of the [R + 1][C] table); the sum runs in physical row order from the
// bias -- exactly live_ring_pass's / live2_stream_ring's order, so v1 = v2 = v3 bit for bit.
// `rings` = the stream's state from ring 1 on (kStateOff[1]): what one bulk-copy stage holds.
template <int I>
MWW_HD void live3_p_taps(const NnWeightsF32 &W, int c, int head, float (&w)[live_ring_rows(I)], float &bias) {
    constexpr int R = live_ring_rows(I), C = live_ring_cols(I);
    const float *taps = (I < 4 ? W.dw_w[I < 4 ? I : 0] : W.head_w) + c;
#pragma unroll
    for (int r = 0; r < R; ++r) { const int j = r < head ? R - head + r : r - head; w[r] = taps[j * C]; }
    bias = I < 4 ? W.dw_b[I < 4 ? I : 0][c] : 0.f;
}
template <int I>
MWW_HD float live3_p_sum(const float *rings, int c, const float (&w)[live_ring_rows(I)], float bias) {
    constexpr int R = live_ring_rows(I), C = live_ring_cols(I);
    constexpr int off = kStateOff[I + 1] - kStateOff[1];
    const float *x = rings + off + c;
    float a = bias;
#pragma unroll
    for (int r = 0; r < R; ++r) a = fmaf(w[r], x[r * C], a);
    return a;
}
// the chain's half of the tail in v3: new first-conv ring = window[120:200], read back from the A operand
MWW_HD void live3_write_ring0(int tid, const float *sm, float *state, long long s0, int n_valid) {
    const int sl = tid >> 3, part = tid & 7;
    if (sl >= n_valid) return;
    const float *a = sm + kLiveOffA;
    for (int k = part; k < 80; k += 8) state[(size_t)(s0 + sl) * kStateFloats + k] = a[(120 + k) * kLivePitch + sl];
}
// after the first conv has consumed A (and a barrier): new first-conv ring = window[120:200], read back from the A operand;
// new pending rows = the call's last n_pend rows, which are NOT part of the window -- read from the caller's rows (only when
// rows are pending at all; the steady state of hop-aligned 30 ms steps has none, so the chain then issues no global load).
// Thread -> (stream = tid / 8, 8 threads per stream)
MWW_HD void live2_write_tail(int tid, const float *sm, const LiveInput &in, float *state, float *pend, long long s0, int n_valid) {
    const int sl = tid >> 3, part = tid & 7;
    if (sl >= n_valid) return;
    const size_t su = (size_t)(s0 + sl);
    const float *a = sm + kLiveOffA;
    for (int k = part; k < 80; k += 8) state[su * (size_t)kStateFloats + k] = a[(120 + k) * kLivePitch + sl];
    const int np40 = in.n_pend * kNumChannels;
    for (int e = part; e < np40; e += 8) pend[su * (size_t)(2 * kNumChannels) + e] = live_row_value(in, su, (unsigned)(3 * kNumChannels - np40 + e));
}

// chain: depthwise of block L (I = L) or head partial (I = 4) from the streamers' P: D = fma(newest tap, x_new, P); the new
// row replaces the oldest physical row of the ring
template <int I>
MWW_HD void live2_dw_from_p(int tid, float *sm, float *state, long long s0, int n_valid, int head, const float *p_buf) {
    constexpr int R = live_ring_rows(I), C = live_ring_cols(I);
    constexpr int per = kLiveStreams * C / kLive2ChainThreads;       // 4 or 8 streams per thread
    constexpr int ring_off = kStateOff[I + 1];
    (void)R;
    const int c = tid % C, sub = tid / C;
    const float wn = sm[kLive2OffSmall + kLive2SmallTaps + live2_col_base(I) + c];
    const float *h = sm + kLiveOffH + c * kLivePitch;
    float *d = sm + kLiveOffD + c * kLivePitch;
    const float *p_col = p_buf + (live2_col_base(I) + c) * kLive2PPitch;
#pragma unroll
    for (int i = 0; i < per; ++i) {
        const int sl = sub * per + i;
        const bool ok = sl < n_valid;
        const float xn = h[sl];
        d[sl] = ok ? fmaf(wn, xn, p_col[sl]) : 0.f;
        if (ok) state[(size_t)(s0 + sl) * kStateFloats + ring_off + head * C + c] = xn;
    }
}

#if defined(__CUDACC__)
// named barriers of the warp-specialised kernel (barrier 0 is __syncthreads)
MWW_D void bar_sync(int id, int count) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); }
MWW_D void bar_arrive(int id, int count) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory"); }

// first conv on tensor cores: 8 warps = 2 stream tiles x 4 channel tiles, K = 200 (25 k-steps), B fragments from L2
MWW_D void live_first_conv_mma(int tid, float *sm, const float *w0, int w0_pitch) {
    const int warp = tid >> 5, lane = tid & 31;
    const int r0 = 16 * (warp >> 2), n0 = 8 * (warp & 3);
    const float *a_base = sm + kLiveOffA;
    float c[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 5
    for (int ks = 0; ks < 25; ++ks) {
        FragA a;
        FragB b;
        load_frag_b(w0, w0_pitch, 8 * ks, n0, lane, b);
        load_frag_a(a_base, kLivePitch, 8 * ks, r0, lane, a);
        mma_tf32(c, a.lo, b.hi);
        mma_tf32(c, a.hi, b.lo);
        mma_tf32(c, a.hi, b.hi);
    }
    live_fc_store_tile(sm, r0, n0, lane, c);
}
// v3: the first conv's B fragments are the same 50 values per thread for every group.  They are loaded (from L2) a layer
// BEFORE they are needed -- while the chain of the previous group is in its head -- so their latency, 2-3x longer while the
// bulk copies saturate the memory system, is off the critical path; `volatile` pins the loads where they are written.
MWW_D void live_first_conv_load_b(int tid, const float *w0, float (&bw)[50]) {
    const int warp = tid >> 5, lane = tid & 31;
    const float *p = w0 + (lane & 3) * 32 + 8 * (warp & 3) + (lane >> 2);
#pragma unroll
    for (int ks = 0; ks < 25; ++ks) {
        asm volatile("ld.global.nc.f32 %0, [%1];" : "=f"(bw[2 * ks]) : "l"(p + (8 * ks) * 32));
        asm volatile("ld.global.nc.f32 %0, [%1];" : "=f"(bw[2 * ks + 1]) : "l"(p + (8 * ks + 4) * 32));
    }
}
MWW_D void live_first_conv_mma_regs(int tid, float *sm, const float (&bw)[50]) {
    const int warp = tid >> 5, lane = tid & 31;
    const int r0 = 16 * (warp >> 2), n0 = 8 * (warp & 3);
    const float *a_base = sm + kLiveOffA;
    float c[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int ks = 0; ks < 25; ++ks) {
        FragA a;
        FragB b;
        split_tf32(bw[2 * ks], b.hi[0], b.lo[0]);
        split_tf32(bw[2 * ks + 1], b.hi[1], b.lo[1]);
        load_frag_a(a_base, kLivePitch, 8 * ks, r0, lane, a);
        mma_tf32(c, a.lo, b.hi);
        mma_tf32(c, a.hi, b.lo);
        mma_tf32(c, a.hi, b.hi);
    }
    live_fc_store_tile(sm, r0, n0, lane, c);
}
// 1x1 of block L: 8 warps = 2 stream tiles x 4 pairs of channel tiles
// SMEM_ALL (v2): block 0's weights and every bias come from shared memory too
template <int L, bool SMEM_ALL = false>
MWW_D void live_pointwise_mma(int tid, float *sm, const NnWeightsF32 &W) {
    constexpr int cin = kGeom[L].cin;
    const int warp = tid >> 5, lane = tid & 31;
    const int r0 = 16 * (warp >> 2), n0 = 16 * (warp & 3);
    const float *d = sm + kLiveOffD;
    const float *wsm = L == 0 ? (SMEM_ALL ? sm + kLive2OffPw0 : W.pw_w[0]) : sm + live_pw_offset<L>();   // v1 block 0: B fragments straight from L2
    constexpr int wld = (L == 0 && !SMEM_ALL) ? 64 : kWLd;
    const float *bias = SMEM_ALL ? sm + kLive2OffSmall + kLive2SmallPwBias + 64 * L : W.pw_b[L];
    float c[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
#pragma unroll 2
    for (int ks = 0; ks < cin / 8; ++ks) {
        FragA a;
        FragB b0, b1;
        load_frag_a(d, kLivePitch, 8 * ks, r0, lane, a);
        load_frag_b(wsm, wld, 8 * ks, n0, lane, b0);
        load_frag_b(wsm, wld, 8 * ks, n0 + 8, lane, b1);
        mma_tf32(c[0], a.lo, b0.hi); mma_tf32(c[1], a.lo, b1.hi);
        mma_tf32(c[0], a.hi, b0.lo); mma_tf32(c[1], a.hi, b1.lo);
        mma_tf32(c[0], a.hi, b0.hi); mma_tf32(c[1], a.hi, b1.hi);
    }
    live_pw_store_tile_b(sm, bias, r0, n0, lane, c[0]);
    live_pw_store_tile_b(sm, bias, r0, n0 + 8, lane, c[1]);
}
#endif

}  // namespace mww
