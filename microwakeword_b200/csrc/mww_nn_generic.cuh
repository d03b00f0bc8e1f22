// mww_nn_generic.cuh -- streaming MixedNet for ANY geometry the reference's builder can emit with its default
// block structure (microwakeword/mixednet.py:278-386: strided first conv, N MixConv blocks = ring-buffered grouped
// depthwise conv + 1x1 pointwise with folded BatchNorm + ReLU, a (head_rows - 1)-row ring, Flatten, Dense(1), sigmoid),
// fp32 and TFLite-int8, with the ring semantics of microwakeword/layers/stream.py:581-595.
//
// The tensor-core kernels (mww_nn_dev.cuh, mww_nn_live.cuh and their int8 twins) are compiled for the okay_nabu geometry
// (notebooks/basic_training_notebook.ipynb:503-509) -- the configuration BASELINE.json measures.  Models trained with
// other --pointwise_filters / --mixconv_kernel_sizes / --first_conv_* / --stride flags take THIS path: the geometry is a
// run-time argument, one CTA owns one stream for the whole call and steps it exactly like the reference's interpreter
// (one model step = `stride` new feature rows), with every ring resident in shared memory as a circular buffer --
// loaded from HBM once per call and written back once, instead of the reference's whole-ring shift per step
// (stream.py:586-590).  CUDA cores only (the contractions of one stream-step are 1 x K x N: nothing for a tensor core),
// plain loads / stores, a barrier between phases: chosen so that tests/host_emul can execute the very same phase functions
// thread by thread on the CPU and compare them with the oracle for several architectures (tests/test_generic_arch.py).
//
// Not supported (mww_create reports MWW_EUNSUPPORTED): residual connections, repeat_in_block > 1, max-pool / spatial
// attention variants (mixednet.py flags that change the graph's topology), first_conv_kernel_size < stride.
#pragma once

#include "mww_nn_i8_dev.cuh"

namespace mww {

constexpr int kGenMaxBlocks = 8;
constexpr int kGenThreads = 128;
constexpr int kGenMaxChannels = 512;
constexpr int kGenMaxKernel = 64;

struct GenArch {
    int c0, k0, stride, n_blocks, head_rows, ring0;       // ring0 = k0 - stride rows kept by the first conv
    int cin[kGenMaxBlocks], cout[kGenMaxBlocks], kmax[kGenMaxBlocks];
    int c_last, max_c;
    // per-stream state (elements; float or int8), oldest row first, [row][channel]: first-conv ring, block rings, head ring
    int st_blk[kGenMaxBlocks], st_head, state_elems;       // the first-conv ring starts at 0
    int pend_cap;                                          // rows of the pending-row buffer: max(stride - 1, 1)
    // shared memory (4-byte elements): window [k0][40], a[max_c], d[max_c], circular rings [kmax][cin], head [head_rows][c_last]
    int sm_win, sm_a, sm_d, sm_blk[kGenMaxBlocks], sm_head, sm_elems;
    long long macs_per_step;
};

// arch tensor of the model container (microwakeword_b200/model_file.py): [c0, k0, stride, 40, n_blocks, head_rows] then
// per block [cout, n_groups, k_1..k_4].  Returns 0 or a negative reason code (-1 malformed, -2 unsupported size).
MWW_HD int gen_arch_from_tensor(const int32_t *a, int n_ints, GenArch *g) {
    if (n_ints < 6) return -1;
    GenArch A = GenArch();
    A.c0 = a[0]; A.k0 = a[1]; A.stride = a[2]; A.n_blocks = a[4]; A.head_rows = a[5];
    if (a[3] != kNumChannels || A.n_blocks < 1 || A.n_blocks > kGenMaxBlocks || n_ints < 6 + 6 * A.n_blocks) return -1;
    if (A.c0 < 1 || A.c0 > kGenMaxChannels || A.k0 < 1 || A.k0 > kGenMaxKernel || A.stride < 1 || A.stride > A.k0 ||
        A.head_rows < 1 || A.head_rows > kGenMaxKernel) return -2;
    A.ring0 = A.k0 - A.stride;
    A.pend_cap = A.stride > 1 ? A.stride - 1 : 1;
    int cin = A.c0, off = A.ring0 * kNumChannels, sm = 0;
    A.max_c = A.c0;
    A.sm_win = sm; sm += A.k0 * kNumChannels;
    long long macs = (long long)A.k0 * kNumChannels * A.c0;
    for (int i = 0; i < A.n_blocks; ++i) {
        const int32_t *e = a + 6 + 6 * i;
        const int cout = e[0], groups = e[1];
        if (cout < 1 || cout > kGenMaxChannels || groups < 1 || groups > 4) return -2;
        int kmax = 0;
        for (int j = 0; j < groups; ++j) { if (e[2 + j] < 1 || e[2 + j] > kGenMaxKernel) return -2; kmax = e[2 + j] > kmax ? e[2 + j] : kmax; }
        A.cin[i] = cin; A.cout[i] = cout; A.kmax[i] = kmax;
        A.st_blk[i] = off; off += (kmax - 1) * cin;
        // MACs as the reference executes them: each MixConv group only has its own taps (mixednet.py:132-136 split)
        int rest = cin;
        for (int j = 0; j < groups; ++j) { const int n = j == 0 ? cin / groups + (cin - cin / groups * groups) : cin / groups; macs += (long long)n * e[2 + j]; rest -= n; }
        (void)rest;
        macs += (long long)cin * cout;
        A.max_c = cout > A.max_c ? cout : A.max_c;
        cin = cout;
    }
    A.c_last = cin;
    A.st_head = off; off += (A.head_rows - 1) * cin;
    A.state_elems = off;
    macs += (long long)A.head_rows * cin;
    A.macs_per_step = macs;
    A.sm_a = sm; sm += A.max_c;
    A.sm_d = sm; sm += A.max_c;
    for (int i = 0; i < A.n_blocks; ++i) { A.sm_blk[i] = sm; sm += A.kmax[i] * A.cin[i]; }
    A.sm_head = sm; sm += A.head_rows * A.c_last;
    A.sm_elems = sm;
    *g = A;
    return 0;
}

struct GenWeightsF32 {
    const float *w0;                                   // [k0][40][c0]
    const float *dw_w[kGenMaxBlocks];                  // [kmax][cin], zero padded at the front for the shorter MixConv kernels
    const float *dw_b[kGenMaxBlocks];                  // [cin]
    const float *pw_w[kGenMaxBlocks];                  // [cin][cout]  BatchNorm folded
    const float *pw_b[kGenMaxBlocks];                  // [cout]
    const float *head_w;                               // [head_rows][c_last]
    const float *head_b;                               // [1]
};

struct GenWeightsI8 {
    const int8_t *w0; const int32_t *b0, *m0, *s0;
    const int8_t *dw_w[kGenMaxBlocks]; const int32_t *dw_b[kGenMaxBlocks], *dw_m[kGenMaxBlocks], *dw_s[kGenMaxBlocks];
    const int8_t *pw_w[kGenMaxBlocks]; const int32_t *pw_b[kGenMaxBlocks], *pw_m[kGenMaxBlocks], *pw_s[kGenMaxBlocks];
    const int8_t *head_w; const int8_t *lut;
    int32_t head_bias, head_mult, head_shift;
    int32_t zp[4 + 2 * kGenMaxBlocks];   // [in, first-conv out, (depthwise out, pointwise out) per block, logit, prob]
    float in_scale;
};

// this call's input of one stream: the virtual row sequence  V = first-conv ring ++ pending rows ++ rows
template <typename T>
struct GenInput {
    const T *state;            // this stream's state (the first-conv ring is its first ring0 rows)
    const T *pend;             // [pend_cap][40]
    int n_pend;
    const void *rows;          // [n_rows][40] uint16 / float32 (/ int8 for a quantised model)
    int n_rows;
    int row_type;              // 0 uint16, 1 float32, 2 int8
};

// ------------------------------------------------------------------------------------------------------------------
// fp32

MWW_HD float gen_virtual_f32(const GenArch &A, const GenInput<float> &in, int v, int f) {
    if (v < A.ring0) return in.state[v * kNumChannels + f];
    v -= A.ring0;
    if (v < in.n_pend) return in.pend[v * kNumChannels + f];
    const long long e = (long long)(v - in.n_pend) * kNumChannels + f;
    if (in.row_type == 1) return static_cast<const float *>(in.rows)[e];
    return (float)static_cast<const uint16_t *>(in.rows)[e] * kFeatureScale;                 // inference.py:93-94
}

// circular ring of block b / the head: slot 0 is the next write position after loading, slots 1.. hold oldest..newest
template <typename T, typename S>
MWW_HD void gen_load_ring(int tid, S *buf, const T *src, int rows_kept, int c) {
    for (int e = tid; e < c; e += kGenThreads) buf[e] = S(0);
    for (int e = tid; e < rows_kept * c; e += kGenThreads) buf[c + e] = (S)src[e];
}
// after the call: `pos` is the next write slot = the oldest row; the kept rows are the kmax - 1 newest, oldest first
template <typename T, typename S>
MWW_HD void gen_store_ring(int tid, const S *buf, T *dst, int slots, int c, int pos) {
    for (int e = tid; e < (slots - 1) * c; e += kGenThreads) {
        const int r = e / c, ch = e - r * c;
        int slot = pos + 1 + r;
        slot = slot >= slots ? slot - slots : slot;
        dst[e] = (T)buf[slot * c + ch];
    }
}

MWW_HD void gen_f32_load_state(int tid, float *sm, const GenArch &A, const float *state) {
    for (int b = 0; b < A.n_blocks; ++b) gen_load_ring(tid, sm + A.sm_blk[b], state + A.st_blk[b], A.kmax[b] - 1, A.cin[b]);
    gen_load_ring(tid, sm + A.sm_head, state + A.st_head, A.head_rows - 1, A.c_last);
}

// phase: the first conv's window of step t = V[stride t .. stride t + k0)
MWW_HD void gen_f32_window(int tid, float *sm, const GenArch &A, const GenInput<float> &in, int t) {
    float *win = sm + A.sm_win;
    for (int e = tid; e < A.k0 * kNumChannels; e += kGenThreads) {
        const int k = e / kNumChannels, f = e - k * kNumChannels;
        win[e] = gen_virtual_f32(A, in, A.stride * t + k, f);
    }
}
// phase: first conv + ReLU (mixednet.py:317-331) -> a[c0]
MWW_HD void gen_f32_first_conv(int tid, float *sm, const GenArch &A, const GenWeightsF32 &W) {
    const float *win = sm + A.sm_win;
    float *a = sm + A.sm_a;
    const int K = A.k0 * kNumChannels;
    for (int o = tid; o < A.c0; o += kGenThreads) {
        float acc = 0.f;
        for (int k = 0; k < K; ++k) acc = fmaf(win[k], W.w0[k * A.c0 + o], acc);
        a[o] = acc > 0.f ? acc : 0.f;
    }
}
// phase: the new row enters block b's ring (stream.py:584-590) and the grouped depthwise conv runs over the last kmax rows
MWW_HD void gen_f32_depthwise(int tid, float *sm, const GenArch &A, const GenWeightsF32 &W, int b, int pos) {
    const int cin = A.cin[b], kmax = A.kmax[b];
    float *buf = sm + A.sm_blk[b];
    const float *a = sm + A.sm_a;
    float *d = sm + A.sm_d;
    for (int c = tid; c < cin; c += kGenThreads) {
        buf[pos * cin + c] = a[c];
        float acc = 0.f;
        int slot = pos + 1;
        for (int j = 0; j < kmax; ++j) {
            slot = slot >= kmax ? slot - kmax : slot;
            acc = fmaf(buf[slot * cin + c], W.dw_w[b][j * cin + c], acc);
            ++slot;
        }
        d[c] = acc + W.dw_b[b][c];
    }
}
// phase: 1x1 projection (BatchNorm folded) + ReLU -> a[cout]
MWW_HD void gen_f32_pointwise(int tid, float *sm, const GenArch &A, const GenWeightsF32 &W, int b) {
    const int cin = A.cin[b], cout = A.cout[b];
    const float *d = sm + A.sm_d;
    float *a = sm + A.sm_a;
    for (int o = tid; o < cout; o += kGenThreads) {
        float acc = 0.f;
        for (int c = 0; c < cin; ++c) acc = fmaf(d[c], W.pw_w[b][c * cout + o], acc);
        acc += W.pw_b[b][o];
        a[o] = acc > 0.f ? acc : 0.f;
    }
}
// phase: head, part 1: the new row enters the head ring; per-channel partial dot products over head_rows rows -> d[c]
MWW_HD void gen_f32_head_partial(int tid, float *sm, const GenArch &A, const GenWeightsF32 &W, int pos) {
    const int cl = A.c_last, hr = A.head_rows;
    float *buf = sm + A.sm_head;
    const float *a = sm + A.sm_a;
    float *d = sm + A.sm_d;
    for (int c = tid; c < cl; c += kGenThreads) {
        buf[pos * cl + c] = a[c];
        float acc = 0.f;
        int slot = pos + 1;
        for (int j = 0; j < hr; ++j) {
            slot = slot >= hr ? slot - hr : slot;
            acc = fmaf(buf[slot * cl + c], W.head_w[j * cl + c], acc);
            ++slot;
        }
        d[c] = acc;
    }
}
// phase: head, part 2 (thread 0): reduce over channels, bias, sigmoid (mixednet.py:383-384)
MWW_HD void gen_f32_head_finish(int tid, const float *sm, const GenArch &A, const GenWeightsF32 &W, float *prob_out) {
    if (tid != 0) return;
    const float *d = sm + A.sm_d;
    float acc = 0.f;
    for (int c = 0; c < A.c_last; ++c) acc += d[c];
    *prob_out = nn_sigmoid(acc + W.head_b[0]);
}
// tail, part 1: the rows the NEXT call starts from -- new first-conv ring = V[sT .. sT + ring0), new pending rows after it --
// are gathered into the (now idle) window buffer while the old ring / pending rows are still intact
MWW_HD void gen_f32_tail_gather(int tid, float *sm, const GenArch &A, const GenInput<float> &in, int n_steps) {
    float *win = sm + A.sm_win;
    const int n_virtual = A.ring0 + in.n_pend + in.n_rows, first = A.stride * n_steps;
    const int n_keep = n_virtual - first;                                   // ring0 + new pending rows  (< k0)
    for (int e = tid; e < n_keep * kNumChannels; e += kGenThreads) {
        const int k = e / kNumChannels, f = e - k * kNumChannels;
        win[e] = gen_virtual_f32(A, in, first + k, f);
    }
}
// tail, part 2 (after a barrier): write everything back
MWW_HD void gen_f32_tail_store(int tid, const float *sm, const GenArch &A, float *state, float *pend, int n_keep, const int *pos /* [n_blocks + 1] */) {
    const float *win = sm + A.sm_win;
    for (int e = tid; e < A.ring0 * kNumChannels; e += kGenThreads) state[e] = win[e];
    for (int e = tid; e < (n_keep - A.ring0) * kNumChannels; e += kGenThreads) pend[e] = win[A.ring0 * kNumChannels + e];
    for (int b = 0; b < A.n_blocks; ++b) gen_store_ring(tid, sm + A.sm_blk[b], state + A.st_blk[b], A.kmax[b], A.cin[b], pos[b]);
    gen_store_ring(tid, sm + A.sm_head, state + A.st_head, A.head_rows, A.c_last, pos[A.n_blocks]);
}

// ------------------------------------------------------------------------------------------------------------------
// int8 (TFLite reference integer kernels, SURVEY.md Appendix C; same arithmetic helpers as mww_nn_i8_dev.cuh).
// Activations live in shared memory as their raw quantised value in an int32.

MWW_HD int32_t gen_virtual_i8(const GenArch &A, const GenWeightsI8 &W, const GenInput<int8_t> &in, int v, int f) {
    if (v < A.ring0) return in.state[v * kNumChannels + f];
    v -= A.ring0;
    if (v < in.n_pend) return in.pend[v * kNumChannels + f];
    const long long e = (long long)(v - in.n_pend) * kNumChannels + f;
    if (in.row_type == 2) return static_cast<const int8_t *>(in.rows)[e];
    const float x = in.row_type == 1 ? static_cast<const float *>(in.rows)[e]
                                     : (float)static_cast<const uint16_t *>(in.rows)[e] * kFeatureScale;
    return nnq_quantize(x, W.in_scale, W.zp[0]);                                              // inference.py:127-147
}
MWW_HD void gen_i8_load_state(int tid, int32_t *sm, const GenArch &A, const int8_t *state) {
    for (int b = 0; b < A.n_blocks; ++b) gen_load_ring(tid, sm + A.sm_blk[b], state + A.st_blk[b], A.kmax[b] - 1, A.cin[b]);
    gen_load_ring(tid, sm + A.sm_head, state + A.st_head, A.head_rows - 1, A.c_last);
}
MWW_HD void gen_i8_window(int tid, int32_t *sm, const GenArch &A, const GenWeightsI8 &W, const GenInput<int8_t> &in, int t) {
    int32_t *win = sm + A.sm_win;
    for (int e = tid; e < A.k0 * kNumChannels; e += kGenThreads) {
        const int k = e / kNumChannels, f = e - k * kNumChannels;
        win[e] = gen_virtual_i8(A, W, in, A.stride * t + k, f);
    }
}
MWW_HD void gen_i8_first_conv(int tid, int32_t *sm, const GenArch &A, const GenWeightsI8 &W) {
    const int32_t *win = sm + A.sm_win;
    int32_t *a = sm + A.sm_a;
    const int K = A.k0 * kNumChannels;
    const int32_t zp_in = W.zp[0], zp_out = W.zp[1];
    for (int o = tid; o < A.c0; o += kGenThreads) {
        int32_t acc = 0;
        for (int k = 0; k < K; ++k) acc += (win[k] - zp_in) * (int32_t)W.w0[k * A.c0 + o];
        acc += W.b0[o];
        a[o] = requant_rel(acc, W.m0[o], W.s0[o], zp_out, true) + zp_out;
    }
}
MWW_HD void gen_i8_depthwise(int tid, int32_t *sm, const GenArch &A, const GenWeightsI8 &W, int b, int pos) {
    const int cin = A.cin[b], kmax = A.kmax[b];
    int32_t *buf = sm + A.sm_blk[b];
    const int32_t *a = sm + A.sm_a;
    int32_t *d = sm + A.sm_d;
    const int32_t zp_in = W.zp[1 + 2 * b], zp_d = W.zp[2 + 2 * b];
    for (int c = tid; c < cin; c += kGenThreads) {
        buf[pos * cin + c] = a[c];
        int32_t acc = 0;
        int slot = pos + 1;
        for (int j = 0; j < kmax; ++j) {
            slot = slot >= kmax ? slot - kmax : slot;
            acc += (buf[slot * cin + c] - zp_in) * (int32_t)W.dw_w[b][j * cin + c];
            ++slot;
        }
        acc += W.dw_b[b][c];
        d[c] = requant_rel(acc, W.dw_m[b][c], W.dw_s[b][c], zp_d, false) + zp_d;
    }
}
MWW_HD void gen_i8_pointwise(int tid, int32_t *sm, const GenArch &A, const GenWeightsI8 &W, int b) {
    const int cin = A.cin[b], cout = A.cout[b];
    const int32_t *d = sm + A.sm_d;
    int32_t *a = sm + A.sm_a;
    const int32_t zp_d = W.zp[2 + 2 * b], zp_p = W.zp[3 + 2 * b];
    for (int o = tid; o < cout; o += kGenThreads) {
        int32_t acc = 0;
        for (int c = 0; c < cin; ++c) acc += (d[c] - zp_d) * (int32_t)W.pw_w[b][c * cout + o];
        acc += W.pw_b[b][o];
        a[o] = requant_rel(acc, W.pw_m[b][o], W.pw_s[b][o], zp_p, true) + zp_p;
    }
}
MWW_HD void gen_i8_head_partial(int tid, int32_t *sm, const GenArch &A, const GenWeightsI8 &W, int pos) {
    const int cl = A.c_last, hr = A.head_rows;
    int32_t *buf = sm + A.sm_head;
    const int32_t *a = sm + A.sm_a;
    int32_t *d = sm + A.sm_d;
    const int32_t zp_in = W.zp[1 + 2 * A.n_blocks];
    for (int c = tid; c < cl; c += kGenThreads) {
        buf[pos * cl + c] = a[c];
        int32_t acc = 0;
        int slot = pos + 1;
        for (int j = 0; j < hr; ++j) {
            slot = slot >= hr ? slot - hr : slot;
            acc += (buf[slot * cl + c] - zp_in) * (int32_t)W.head_w[j * cl + c];
            ++slot;
        }
        d[c] = acc;
    }
}
// FULLY_CONNECTED requant -> LOGISTIC LUT -> QUANTIZE to uint8 -> Model.dequantize_output_data (/255, inference.py:162-170)
MWW_HD void gen_i8_head_finish(int tid, const int32_t *sm, const GenArch &A, const GenWeightsI8 &W, float *prob_out) {
    if (tid != 0) return;
    const int32_t *d = sm + A.sm_d;
    int32_t acc = 0;
    for (int c = 0; c < A.c_last; ++c) acc += d[c];
    acc += W.head_bias;
    const int32_t zp_fc = W.zp[2 + 2 * A.n_blocks];
    const int32_t logit = requant_rel(acc, W.head_mult, W.head_shift, zp_fc, false) + zp_fc;
    const int out_u8 = (int)W.lut[(uint8_t)(int8_t)logit] + 128;
    *prob_out = (1.0f / 255.0f) * (float)out_u8;
}
MWW_HD void gen_i8_tail_gather(int tid, int32_t *sm, const GenArch &A, const GenWeightsI8 &W, const GenInput<int8_t> &in, int n_steps) {
    int32_t *win = sm + A.sm_win;
    const int n_virtual = A.ring0 + in.n_pend + in.n_rows, first = A.stride * n_steps;
    const int n_keep = n_virtual - first;
    for (int e = tid; e < n_keep * kNumChannels; e += kGenThreads) {
        const int k = e / kNumChannels, f = e - k * kNumChannels;
        win[e] = gen_virtual_i8(A, W, in, first + k, f);
    }
}
MWW_HD void gen_i8_tail_store(int tid, const int32_t *sm, const GenArch &A, int8_t *state, int8_t *pend, int n_keep, const int *pos) {
    const int32_t *win = sm + A.sm_win;
    for (int e = tid; e < A.ring0 * kNumChannels; e += kGenThreads) state[e] = (int8_t)win[e];
    for (int e = tid; e < (n_keep - A.ring0) * kNumChannels; e += kGenThreads) pend[e] = (int8_t)win[A.ring0 * kNumChannels + e];
    for (int b = 0; b < A.n_blocks; ++b) gen_store_ring(tid, sm + A.sm_blk[b], state + A.st_blk[b], A.kmax[b], A.cin[b], pos[b]);
    gen_store_ring(tid, sm + A.sm_head, state + A.st_head, A.head_rows, A.c_last, pos[A.n_blocks]);
}
// reset value of one element of the state / pending buffers: the zero point of the tensor the ring buffers
// (quantised state variables hold real 0, utils.py:333)
MWW_HD int8_t gen_i8_reset_value(const GenArch &A, const GenWeightsI8 &W, int e /* index into the state */) {
    if (e < A.ring0 * kNumChannels) return (int8_t)W.zp[0];
    for (int b = A.n_blocks - 1; b >= 0; --b)
        if (e >= A.st_blk[b] && e < A.st_blk[b] + (A.kmax[b] - 1) * A.cin[b]) return (int8_t)W.zp[1 + 2 * b];
    return (int8_t)W.zp[1 + 2 * A.n_blocks];
}

// ------------------------------------------------------------------------------------------------------------------
// hybrid: the float graph of a model converted with dynamic-range quantisation (utils.py:328 without a representative
// dataset).  Large CONV_2D / DEPTHWISE_CONV_2D / FULLY_CONNECTED ops carry symmetric per-channel int8 weights, and TFLite's
// hybrid kernels quantise the op's whole float input tensor to int8 on every invoke, accumulate int8 x int8 in int32 and
// rescale to float.  Activations and rings stay fp32 in the fp32 state layout; float ops of such a model run the fp32
// phases above.  Arithmetic: tests/hybrid_ref/hybrid_ref.c [UPSTREAM-RECALL], reproduced operation for operation -- the rescales use
// round-to-nearest intrinsics so that nvcc cannot contract them into an FMA, because a one-ulp difference before a
// quantiser flips an int8 code.
//
// One hybrid op = four phases: min/max partials of its input tensor (per thread), the scale / zero point (one thread per
// quantiser, in double precision), quantisation into an int8 buffer, then int32 dot products and the float epilogue.

constexpr int kHyFloat = 0, kHyAsymmetric = 1, kHySymmetric = 2;     // hy/mode entries (model_file.py)
constexpr int kHyMaxQ = 4;                                              // quantisers in flight: the MixConv groups of a block

struct GenHybrid {
    int mode0, mode_head;
    int mode_pw[kGenMaxBlocks], any_dw[kGenMaxBlocks], n_groups[kGenMaxBlocks];
    int g_k[kGenMaxBlocks][kHyMaxQ], g_c0[kGenMaxBlocks][kHyMaxQ], g_n[kGenMaxBlocks][kHyMaxQ], g_mode[kGenMaxBlocks][kHyMaxQ];
    const int8_t *w0; const float *s0;                                   // [k0][40][c0], [c0]
    const int8_t *dw_w[kGenMaxBlocks]; const float *dw_s[kGenMaxBlocks]; // [kmax][cin] (0 in float groups), [cin]
    const int8_t *pw_w[kGenMaxBlocks]; const float *pw_s[kGenMaxBlocks]; // [cin][cout], [cout]
    const int8_t *head_w; const float *head_s;                           // [head_rows][c_last], [1]
    // shared memory past GenArch::sm_elems (4-byte elements): quantiser parameters [kHyMaxQ][4] (scale, 1/scale, zero point),
    // min/max partials [kHyMaxQ][2][kGenThreads], int8 codes of one op's input
    int sm_par, sm_red, sm_q, sm_elems;
};

// modes = hy/mode (model_file.hybrid_slots order).  Returns 0, or -1 when the vector does not fit the architecture.
MWW_HD int gen_hybrid_layout(const GenArch &A, const int32_t *arch, const int32_t *modes, int n_modes, GenHybrid *H) {
    int s = 0, q_bytes = A.k0 * kNumChannels;
    if (n_modes < 2) return -1;
    H->mode0 = modes[s++];
    for (int b = 0; b < A.n_blocks; ++b) {
        const int32_t *e = arch + 6 + 6 * b;
        const int groups = e[1];
        H->n_groups[b] = groups;
        H->any_dw[b] = 0;
        int c = 0;
        for (int j = 0; j < groups; ++j) {
            if (s >= n_modes) return -1;
            H->g_k[b][j] = e[2 + j];
            H->g_n[b][j] = A.cin[b] / groups + (j == 0 ? A.cin[b] % groups : 0);      // mixednet.py:132-136
            H->g_c0[b][j] = c; c += H->g_n[b][j];
            H->g_mode[b][j] = modes[s++];
            H->any_dw[b] |= H->g_mode[b][j] != kHyFloat;
        }
        if (s >= n_modes) return -1;
        H->mode_pw[b] = modes[s++];
        q_bytes = A.kmax[b] * A.cin[b] > q_bytes ? A.kmax[b] * A.cin[b] : q_bytes;
    }
    if (s >= n_modes) return -1;
    H->mode_head = modes[s++];
    if (s != n_modes) return -1;
    for (int i = 0; i < n_modes; ++i) if (modes[i] < kHyFloat || modes[i] > kHySymmetric) return -1;
    q_bytes = A.head_rows * A.c_last > q_bytes ? A.head_rows * A.c_last : q_bytes;
    q_bytes = A.max_c > q_bytes ? A.max_c : q_bytes;
    int sm = A.sm_elems;
    H->sm_par = sm; sm += 4 * kHyMaxQ;
    H->sm_red = sm; sm += 2 * kHyMaxQ * kGenThreads;
    H->sm_q = sm; sm += (q_bytes + 3) / 4;
    H->sm_elems = sm;
    return 0;
}

MWW_HD float hy_mul(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}
MWW_HD float hy_add(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fadd_rn(a, b);
#else
    return a + b;
#endif
}
MWW_HD float hy_div(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fdiv_rn(a, b);
#else
    return a / b;
#endif
}
MWW_HD double hy_dsub(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dsub_rn(a, b);
#else
    return a - b;
#endif
}
MWW_HD double hy_ddiv(double a, double b) {
#ifdef __CUDA_ARCH__
    return __ddiv_rn(a, b);
#else
    return a / b;
#endif
}
MWW_HD double hy_dadd(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}

MWW_HD void hy_put_partial(float *sm, const GenHybrid &H, int q, int tid, float mn, float mx) {
    sm[H.sm_red + (2 * q) * kGenThreads + tid] = mn;
    sm[H.sm_red + (2 * q + 1) * kGenThreads + tid] = mx;
}

// phase: thread q finishes quantiser q; `mode` is that quantiser's mode (kHyFloat: none for this thread).  Exact min / max of
// the partials, then AsymmetricQuantizeFloats' scale and nudged zero point in double / SymmetricQuantizeFloats' range
MWW_HD void gen_hy_qparams(int tid, float *sm, const GenHybrid &H, int mode) {
    if (tid >= kHyMaxQ || mode == kHyFloat) return;
    const float *pmn = sm + H.sm_red + (2 * tid) * kGenThreads, *pmx = pmn + kGenThreads;
    float mn = pmn[0], mx = pmx[0];
    for (int i = 1; i < kGenThreads; ++i) { mn = pmn[i] < mn ? pmn[i] : mn; mx = pmx[i] > mx ? pmx[i] : mx; }
    float *par = sm + H.sm_par + 4 * tid;
    if (mode == kHySymmetric) {
        const float range = fmaxf(fabsf(mn), fabsf(mx));
        if (range == 0.0f) { par[0] = 1.0f; par[1] = 0.0f; par[2] = 0.0f; return; }
        par[0] = hy_div(range, 127.0f); par[1] = hy_div(127.0f, range); par[2] = 0.0f;
        return;
    }
    const double rmin = fmin(0.0, (double)mn), rmax = fmax(0.0, (double)mx);
    if (rmin == rmax) { par[0] = 1.0f; par[1] = 0.0f; par[2] = 0.0f; return; }
    const double qmin = -128.0, qmax = 127.0;
    const double scale = hy_ddiv(hy_dsub(rmax, rmin), 255.0);
    const double zp_from_min = hy_dsub(qmin, hy_ddiv(rmin, scale)), zp_from_max = hy_dsub(qmax, hy_ddiv(rmax, scale));
    const double err_min = hy_dadd(fabs(qmin), fabs(hy_ddiv(rmin, scale))), err_max = hy_dadd(fabs(qmax), fabs(hy_ddiv(rmax, scale)));
    const double zp_d = err_min < err_max ? zp_from_min : zp_from_max;
    const float zp = zp_d <= qmin ? -128.0f : (zp_d >= qmax ? 127.0f : (float)round(zp_d));
    const float sf = (float)scale;
    par[0] = sf; par[1] = hy_div(1.0f, sf); par[2] = zp;
}

// one element of quantiser q (the all-zero case has 1/scale 0 and zero point 0, so it yields code 0 like the reference)
MWW_HD int32_t hy_code(const float *par, int mode, float x) {
    if (mode == kHySymmetric) {
        const int32_t v = (int32_t)roundf(hy_mul(x, par[1]));
        return v < -127 ? -127 : (v > 127 ? 127 : v);
    }
    const int32_t v = (int32_t)roundf(hy_add(par[2], hy_mul(x, par[1])));
    return v < -128 ? -128 : (v > 127 ? 127 : v);
}

// CONV_2D / DEPTHWISE_CONV_2D per-channel epilogue: (float)acc * w_scale * input_scale + bias, left to right
MWW_HD float hy_conv_out(int32_t acc, float w_scale, float in_scale, float bias) {
    return hy_add(hy_mul(hy_mul((float)acc, w_scale), in_scale), bias);
}

// ---- first conv: the [k0, 40] window is the op's input tensor
// phase: window (as gen_f32_window) + min / max partials
MWW_HD void gen_hy_window(int tid, float *sm, const GenArch &A, const GenHybrid &H, const GenInput<float> &in, int t) {
    float *win = sm + A.sm_win;
    float mn = INFINITY, mx = -INFINITY;
    for (int e = tid; e < A.k0 * kNumChannels; e += kGenThreads) {
        const int k = e / kNumChannels, f = e - k * kNumChannels;
        const float v = gen_virtual_f32(A, in, A.stride * t + k, f);
        win[e] = v;
        mn = v < mn ? v : mn; mx = v > mx ? v : mx;
    }
    hy_put_partial(sm, H, 0, tid, mn, mx);
}
MWW_HD void gen_hy_quant_window(int tid, float *sm, const GenArch &A, const GenHybrid &H) {
    const float *win = sm + A.sm_win, *par = sm + H.sm_par;
    int8_t *q = reinterpret_cast<int8_t *>(sm + H.sm_q);
    for (int e = tid; e < A.k0 * kNumChannels; e += kGenThreads) q[e] = (int8_t)hy_code(par, H.mode0, win[e]);
}
MWW_HD void gen_hy_first_conv(int tid, float *sm, const GenArch &A, const GenHybrid &H) {
    const int8_t *q = reinterpret_cast<const int8_t *>(sm + H.sm_q);
    const float *par = sm + H.sm_par;
    float *a = sm + A.sm_a;
    const int K = A.k0 * kNumChannels;
    const int32_t zp = (int32_t)par[2];
    for (int o = tid; o < A.c0; o += kGenThreads) {
        int32_t acc = 0;
        for (int k = 0; k < K; ++k) acc += ((int32_t)q[k] - zp) * (int32_t)H.w0[k * A.c0 + o];
        const float y = hy_conv_out(acc, H.s0[o], par[0], 0.0f);
        a[o] = y > 0.f ? y : 0.f;
    }
}

// ---- MixConv block with at least one hybrid group; group g's input tensor = the LAST k_g rows of the ring memory in its
// channels (StridedKeep).  After the insert the newest row sits in slot pos; "age" 0 = newest.
MWW_HD int hy_group_of(const GenHybrid &H, int b, int c) {
    int g = 0;
    while (g + 1 < H.n_groups[b] && c >= H.g_c0[b][g + 1]) ++g;
    return g;
}
// element i of group g's input tensor [k_g][n_g] -> ring slot (row r = i / n_g, oldest first) and channel
MWW_HD void hy_group_elem(const GenArch &A, const GenHybrid &H, int b, int g, int pos, int i, int *slot, int *c, int *age) {
    const int n = H.g_n[b][g], r = i / n;
    *c = H.g_c0[b][g] + (i - r * n);
    *age = H.g_k[b][g] - 1 - r;
    const int sl = pos - *age;
    *slot = sl < 0 ? sl + A.kmax[b] : sl;
}
// phase: the new row enters the ring + min / max partials of every hybrid group (the newest row is read from a[])
MWW_HD void gen_hy_block_insert(int tid, float *sm, const GenArch &A, const GenHybrid &H, int b, int pos) {
    const int cin = A.cin[b];
    float *buf = sm + A.sm_blk[b];
    const float *a = sm + A.sm_a;
    for (int c = tid; c < cin; c += kGenThreads) buf[pos * cin + c] = a[c];
    for (int g = 0; g < H.n_groups[b]; ++g) {
        if (H.g_mode[b][g] == kHyFloat) continue;
        float mn = INFINITY, mx = -INFINITY;
        for (int i = tid; i < H.g_k[b][g] * H.g_n[b][g]; i += kGenThreads) {
            int slot, c, age;
            hy_group_elem(A, H, b, g, pos, i, &slot, &c, &age);
            const float v = age == 0 ? a[c] : buf[slot * cin + c];
            mn = v < mn ? v : mn; mx = v > mx ? v : mx;
        }
        hy_put_partial(sm, H, g, tid, mn, mx);
    }
}
MWW_HD void gen_hy_quant_block(int tid, float *sm, const GenArch &A, const GenHybrid &H, int b, int pos) {
    const int cin = A.cin[b];
    const float *buf = sm + A.sm_blk[b];
    int8_t *q = reinterpret_cast<int8_t *>(sm + H.sm_q);
    for (int g = 0; g < H.n_groups[b]; ++g) {
        if (H.g_mode[b][g] == kHyFloat) continue;
        const float *par = sm + H.sm_par + 4 * g;
        for (int i = tid; i < H.g_k[b][g] * H.g_n[b][g]; i += kGenThreads) {
            int slot, c, age;
            hy_group_elem(A, H, b, g, pos, i, &slot, &c, &age);
            q[slot * cin + c] = (int8_t)hy_code(par, H.g_mode[b][g], buf[slot * cin + c]);
        }
    }
}
// phase: grouped depthwise conv -> d[cin]; hybrid groups in int32 over their own k taps, float groups as gen_f32_depthwise
MWW_HD void gen_hy_depthwise(int tid, float *sm, const GenArch &A, const GenWeightsF32 &W, const GenHybrid &H, int b, int pos) {
    const int cin = A.cin[b], kmax = A.kmax[b];
    const float *buf = sm + A.sm_blk[b];
    const int8_t *q = reinterpret_cast<const int8_t *>(sm + H.sm_q);
    float *d = sm + A.sm_d;
    for (int c = tid; c < cin; c += kGenThreads) {
        const int g = hy_group_of(H, b, c);
        if (H.g_mode[b][g] == kHyFloat) {
            float acc = 0.f;
            int slot = pos + 1;
            for (int j = 0; j < kmax; ++j) {
                slot = slot >= kmax ? slot - kmax : slot;
                acc = fmaf(buf[slot * cin + c], W.dw_w[b][j * cin + c], acc);
                ++slot;
            }
            d[c] = acc + W.dw_b[b][c];
            continue;
        }
        const float *par = sm + H.sm_par + 4 * g;
        const int32_t zp = (int32_t)par[2];
        const int k = H.g_k[b][g];
        int slot = pos - (k - 1);
        slot = slot < 0 ? slot + kmax : slot;
        int32_t acc = 0;
        for (int r = 0; r < k; ++r) {
            acc += ((int32_t)q[slot * cin + c] - zp) * (int32_t)H.dw_w[b][(kmax - k + r) * cin + c];
            slot = slot + 1 == kmax ? 0 : slot + 1;
        }
        d[c] = hy_conv_out(acc, H.dw_s[b][c], par[0], W.dw_b[b][c]);
    }
}

// ---- hybrid 1x1 conv: the op's input tensor is d[cin]
MWW_HD void gen_hy_minmax_d(int tid, float *sm, const GenArch &A, const GenHybrid &H, int b) {
    const float *d = sm + A.sm_d;
    float mn = INFINITY, mx = -INFINITY;
    for (int c = tid; c < A.cin[b]; c += kGenThreads) { mn = d[c] < mn ? d[c] : mn; mx = d[c] > mx ? d[c] : mx; }
    hy_put_partial(sm, H, 0, tid, mn, mx);
}
MWW_HD void gen_hy_quant_d(int tid, float *sm, const GenArch &A, const GenHybrid &H, int b) {
    const float *d = sm + A.sm_d, *par = sm + H.sm_par;
    int8_t *q = reinterpret_cast<int8_t *>(sm + H.sm_q);
    for (int c = tid; c < A.cin[b]; c += kGenThreads) q[c] = (int8_t)hy_code(par, H.mode_pw[b], d[c]);
}
MWW_HD void gen_hy_pointwise(int tid, float *sm, const GenArch &A, const GenWeightsF32 &W, const GenHybrid &H, int b) {
    const int cin = A.cin[b], cout = A.cout[b];
    const int8_t *q = reinterpret_cast<const int8_t *>(sm + H.sm_q);
    const float *par = sm + H.sm_par;
    float *a = sm + A.sm_a;
    const int32_t zp = (int32_t)par[2];
    for (int o = tid; o < cout; o += kGenThreads) {
        int32_t acc = 0;
        for (int c = 0; c < cin; ++c) acc += ((int32_t)q[c] - zp) * (int32_t)H.pw_w[b][c * cout + o];
        const float y = hy_conv_out(acc, H.pw_s[b][o], par[0], W.pw_b[b][o]);
        a[o] = y > 0.f ? y : 0.f;
    }
}

// ---- hybrid dense head: the op's input tensor is the whole [head_rows, c_last] ring memory
MWW_HD void gen_hy_head_insert(int tid, float *sm, const GenArch &A, const GenHybrid &H, int pos) {
    const int cl = A.c_last, hr = A.head_rows;
    float *buf = sm + A.sm_head;
    const float *a = sm + A.sm_a;
    float mn = INFINITY, mx = -INFINITY;
    for (int c = tid; c < cl; c += kGenThreads) buf[pos * cl + c] = a[c];
    for (int e = tid; e < hr * cl; e += kGenThreads) {
        const int slot = e / cl, c = e - slot * cl;
        const float v = slot == pos ? a[c] : buf[e];
        mn = v < mn ? v : mn; mx = v > mx ? v : mx;
    }
    hy_put_partial(sm, H, 0, tid, mn, mx);
}
MWW_HD void gen_hy_quant_head(int tid, float *sm, const GenArch &A, const GenHybrid &H) {
    const float *buf = sm + A.sm_head, *par = sm + H.sm_par;
    int8_t *q = reinterpret_cast<int8_t *>(sm + H.sm_q);
    for (int e = tid; e < A.head_rows * A.c_last; e += kGenThreads) q[e] = (int8_t)hy_code(par, H.mode_head, buf[e]);
}
// per-channel int32 partial sums over the rows, stored in d[c] as floats (|partial| <= 64 * 255 * 128 < 2^24: exact)
MWW_HD void gen_hy_head_partial(int tid, float *sm, const GenArch &A, const GenHybrid &H, int pos) {
    const int cl = A.c_last, hr = A.head_rows;
    const int8_t *q = reinterpret_cast<const int8_t *>(sm + H.sm_q);
    const int32_t zp = (int32_t)sm[H.sm_par + 2];
    float *d = sm + A.sm_d;
    for (int c = tid; c < cl; c += kGenThreads) {
        int32_t acc = 0;
        int slot = pos + 1;
        for (int j = 0; j < hr; ++j) {
            slot = slot >= hr ? slot - hr : slot;
            acc += ((int32_t)q[slot * cl + c] - zp) * (int32_t)H.head_w[j * cl + c];
            ++slot;
        }
        d[c] = (float)acc;
    }
}
// tail, part 2: as gen_f32_tail_store; after n_steps steps from slot 0 the next write slot of a ring of R slots is n_steps % R
MWW_HD void gen_hy_tail_store(int tid, const float *sm, const GenArch &A, float *state, float *pend, int n_keep, int n_steps) {
    const float *win = sm + A.sm_win;
    for (int e = tid; e < A.ring0 * kNumChannels; e += kGenThreads) state[e] = win[e];
    for (int e = tid; e < (n_keep - A.ring0) * kNumChannels; e += kGenThreads) pend[e] = win[A.ring0 * kNumChannels + e];
    for (int b = 0; b < A.n_blocks; ++b) gen_store_ring(tid, sm + A.sm_blk[b], state + A.st_blk[b], A.kmax[b], A.cin[b], n_steps % A.kmax[b]);
    gen_store_ring(tid, sm + A.sm_head, state + A.st_head, A.head_rows, A.c_last, n_steps % A.head_rows);
}
// FULLY_CONNECTED: bias + (float)acc * (input_scale * weight_scale), then LOGISTIC in float (thread 0)
MWW_HD void gen_hy_head_finish(int tid, const float *sm, const GenArch &A, const GenWeightsF32 &W, const GenHybrid &H, float *prob_out) {
    if (tid != 0) return;
    const float *d = sm + A.sm_d;
    int32_t acc = 0;
    for (int c = 0; c < A.c_last; ++c) acc += (int32_t)d[c];
    const float logit = hy_add(W.head_b[0], hy_mul((float)acc, hy_mul(sm[H.sm_par], H.head_s[0])));
    *prob_out = nn_sigmoid(logit);
}

}  // namespace mww
