// tests/host_emul/emul_nn.cc -- TEST INFRASTRUCTURE: CPU execution of the product's fp32 MixedNet phase
// functions (microwakeword_b200/csrc/mww_nn_dev.cuh), barriers modelled as phase boundaries.
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "../../microwakeword_b200/csrc/mww_nn_live.cuh"

using namespace mww;


// ---- host model of mma.sync.m16n8k8.tf32 for one warp (fragment layouts from the PTX ISA) -------------
namespace {
float tf32_of(uint32_t bits) { bits &= 0xFFFFE000u; float f; memcpy(&f, &bits, 4); return f; }   // hardware ignores the low 13 bits

void warp_mma_tf32(float (*c)[4], const uint32_t (*a)[4], const uint32_t (*b)[2]) {
    float A[16][8], B[8][8], C[16][8];
    for (int lane = 0; lane < 32; ++lane) {
        const int g = lane >> 2, tig = lane & 3;
        A[g][tig] = tf32_of(a[lane][0]); A[g + 8][tig] = tf32_of(a[lane][1]);
        A[g][tig + 4] = tf32_of(a[lane][2]); A[g + 8][tig + 4] = tf32_of(a[lane][3]);
        B[tig][g] = tf32_of(b[lane][0]); B[tig + 4][g] = tf32_of(b[lane][1]);
        C[g][2 * tig] = c[lane][0]; C[g][2 * tig + 1] = c[lane][1];
        C[g + 8][2 * tig] = c[lane][2]; C[g + 8][2 * tig + 1] = c[lane][3];
    }
    for (int m = 0; m < 16; ++m)
        for (int n = 0; n < 8; ++n) {
            float acc = C[m][n];
            for (int k = 0; k < 8; ++k) acc += A[m][k] * B[k][n];
            C[m][n] = acc;
        }
    for (int lane = 0; lane < 32; ++lane) {
        const int g = lane >> 2, tig = lane & 3;
        c[lane][0] = C[g][2 * tig]; c[lane][1] = C[g][2 * tig + 1];
        c[lane][2] = C[g + 8][2 * tig]; c[lane][3] = C[g + 8][2 * tig + 1];
    }
}

void warp_mma_3xtf32(float (*c)[4], const FragA *a, const FragB *b) {
    uint32_t ah[32][4], al[32][4], bh[32][2], bl[32][2];
    for (int l = 0; l < 32; ++l) {
        for (int i = 0; i < 4; ++i) { ah[l][i] = a[l].hi[i]; al[l][i] = a[l].lo[i]; }
        for (int i = 0; i < 2; ++i) { bh[l][i] = b[l].hi[i]; bl[l][i] = b[l].lo[i]; }
    }
    warp_mma_tf32(c, al, bh);
    warp_mma_tf32(c, ah, bl);
    warp_mma_tf32(c, ah, bh);
}

template <int L>
void emul_pointwise_mma(float *sm, const NnWeightsF32 &W) {
    constexpr int cin = kGeom[L].cin;
    for (int warp = 0; warp < kNnThreads / 32; ++warp) {
        const int t0 = 16 * pw_m_tile(warp), nt0 = pw_n_first(warp), ntc = pw_n_count(warp);
        const float *d = sm + kXFloats;
        const float *wsm = nn_pw_weight_buffer<L>(sm);
        float c[3][32][4] = {};
        for (int ks = 0; ks < cin / 8; ++ks) {
            FragA a[32];
            for (int lane = 0; lane < 32; ++lane) load_frag_a_d(d, 8 * ks, t0, lane, a[lane]);
            for (int i = 0; i < ntc; ++i) {
                FragB b[32];
                for (int lane = 0; lane < 32; ++lane) load_frag_b(wsm, kWLd, 8 * ks, 8 * (nt0 + i), lane, b[lane]);
                warp_mma_3xtf32(c[i], a, b);
            }
        }
        for (int i = 0; i < ntc; ++i)
            for (int lane = 0; lane < 32; ++lane) pw_store_tile<L>(sm, W, t0, 8 * (nt0 + i), lane, c[i][lane]);
    }
}

void emul_first_conv_mma(float *sm, const NnWeightsF32 &W) {
    const float *feat = sm + kXFloats + kDFloats;
    static float c[kNnThreads / 32][4][32][4];
    memset(c, 0, sizeof c);
    for (int warp = 0; warp < kNnThreads / 32; ++warp) {        // part a
        const int t0 = 16 * fc_m_tile(warp);
        for (int ks = fc_k_begin(warp); ks < fc_k_end(warp); ++ks) {
            FragA a[32];
            for (int lane = 0; lane < 32; ++lane) fc_load_frag_a(feat, ks, t0, lane, a[lane]);
            for (int i = 0; i < 4; ++i) {
                FragB b[32];
                for (int lane = 0; lane < 32; ++lane) fc_load_frag_b(W.w0, ks, 8 * i, lane, b[lane]);
                warp_mma_3xtf32(c[warp][i], a, b);
            }
        }
        if (warp % 3 > 0)
            for (int i = 0; i < 4; ++i)
                for (int lane = 0; lane < 32; ++lane) fc_store_partial(sm, warp % 3, t0, 8 * i, lane, c[warp][i][lane]);
    }
    for (int warp = 0; warp < kNnThreads / 32; ++warp) {        // part b, after the barrier
        if (warp % 3 != 0) continue;
        for (int i = 0; i < 4; ++i)
            for (int lane = 0; lane < 32; ++lane) fc_finish_tile(sm, 16 * fc_m_tile(warp), 8 * i, lane, c[warp][i][lane]);
    }
}
}  // namespace

extern "C" int emul_nn_f32(const float *const *wp /* w0, dw_w[4], dw_b[4], pw_w[4], pw_b[4], head_w, head_b */,
                           float *state, float *pend, int n_pend, const void *rows, int n_rows, int rows_are_f32,
                           int n_streams, float *probs, int max_probs, float *logits) {
    NnWeightsF32 W;
    W.w0 = wp[0];
    for (int i = 0; i < 4; ++i) { W.dw_w[i] = wp[1 + i]; W.dw_b[i] = wp[5 + i]; W.pw_w[i] = wp[9 + i]; W.pw_b[i] = wp[13 + i]; }
    W.head_w = wp[17];
    W.head_b = wp[18];
    const int n_virtual = n_pend + n_rows;
    const int n_steps = n_virtual / 3;
    const size_t row_bytes = (size_t)kNumChannels * (rows_are_f32 ? 4 : 2);
    std::vector<float> smv(kNnSmemFloats);
    float *sm = smv.data();
    for (int s = 0; s < n_streams; ++s) {
        for (auto &v : smv) v = -1234.5f;   // poison
        float *my_state = state + (size_t)s * kStateFloats;
        float *my_pend = pend + (size_t)s * 2 * kNumChannels;
        NnInput in;
        in.ring0 = my_state; in.pend = my_pend; in.n_pend = n_pend;
        in.rows = static_cast<const char *>(rows) + (size_t)s * n_rows * row_bytes;
        in.n_rows = n_rows; in.rows_are_f32 = rows_are_f32;
#define ALL(stmt) for (int tid = 0; tid < kNnThreads; ++tid) { stmt; }
        ALL(nn_load_state(tid, sm, my_state));
        for (int step0 = 0; step0 < n_steps; step0 += kTT) {
            const int n = n_steps - step0 < kTT ? n_steps - step0 : kTT;
            ALL(nn_load_features(tid, sm, in, step0, n));
            emul_first_conv_mma(sm, W);
            ALL(nn_stage_pw_weights<0>(tid, sm, W)); ALL(nn_stage_pw_weights<1>(tid, sm, W));
            ALL(nn_depthwise<0>(tid, sm, W)); emul_pointwise_mma<0>(sm, W);
            ALL(nn_stage_pw_weights<2>(tid, sm, W));
            ALL(nn_depthwise<1>(tid, sm, W)); emul_pointwise_mma<1>(sm, W);
            ALL(nn_stage_pw_weights<3>(tid, sm, W));
            ALL(nn_depthwise<2>(tid, sm, W)); emul_pointwise_mma<2>(sm, W);
            ALL(nn_depthwise<3>(tid, sm, W)); emul_pointwise_mma<3>(sm, W);
            ALL(nn_head_partial(tid, sm, W));
            ALL(nn_head_finish(tid, sm, W, n, probs + (size_t)s * max_probs + step0, logits ? logits + (size_t)s * max_probs + step0 : nullptr));
            std::vector<float> tmp((size_t)kNnThreads * 5 * kShiftPerThread);
            ALL(nn_shift_read(tid, sm, n, *reinterpret_cast<float(*)[5][kShiftPerThread]>(&tmp[(size_t)tid * 5 * kShiftPerThread])));
            ALL(nn_shift_write(tid, sm, *reinterpret_cast<float(*)[5][kShiftPerThread]>(&tmp[(size_t)tid * 5 * kShiftPerThread])));
        }
        std::vector<NnTail> tails(kNnThreads);
        ALL(nn_tail_read(tid, in, n_steps, n_virtual, tails[tid]));
        ALL(nn_tail_write(tid, sm, my_state, my_pend, tails[tid]));
#undef ALL
    }
    return n_steps;
}

// ---- int8 path --------------------------------------------------------------------------------
#include "../../microwakeword_b200/csrc/mww_nn_i8_prep.h"


// ---- host model of mma.sync.m16n8k32.s8 for one warp ------------------------------------------------------
namespace {
void warp_mma_s8(int32_t (*c)[4], const FragA8 *a, const FragB8 *b) {
    int32_t A[16][32], B[32][8], C[16][8];
    for (int lane = 0; lane < 32; ++lane) {
        const int g = lane >> 2, tig = lane & 3;
        for (int i = 0; i < 4; ++i) {
            A[g][4 * tig + i] = (int8_t)(a[lane].r[0] >> (8 * i)); A[g + 8][4 * tig + i] = (int8_t)(a[lane].r[1] >> (8 * i));
            A[g][16 + 4 * tig + i] = (int8_t)(a[lane].r[2] >> (8 * i)); A[g + 8][16 + 4 * tig + i] = (int8_t)(a[lane].r[3] >> (8 * i));
            B[4 * tig + i][g] = (int8_t)(b[lane].r[0] >> (8 * i)); B[16 + 4 * tig + i][g] = (int8_t)(b[lane].r[1] >> (8 * i));
        }
        C[g][2 * tig] = c[lane][0]; C[g][2 * tig + 1] = c[lane][1]; C[g + 8][2 * tig] = c[lane][2]; C[g + 8][2 * tig + 1] = c[lane][3];
    }
    for (int m = 0; m < 16; ++m)
        for (int n = 0; n < 8; ++n) { int32_t acc = C[m][n]; for (int k = 0; k < 32; ++k) acc += A[m][k] * B[k][n]; C[m][n] = acc; }
    for (int lane = 0; lane < 32; ++lane) {
        const int g = lane >> 2, tig = lane & 3;
        c[lane][0] = C[g][2 * tig]; c[lane][1] = C[g][2 * tig + 1]; c[lane][2] = C[g + 8][2 * tig]; c[lane][3] = C[g + 8][2 * tig + 1];
    }
}

void emul_q_first_conv_mma(int32_t *sm, const NnWeightsI8 &W) {
    const int8_t *a8 = nnq_bytes(sm) + kQOffA8, *w0 = nnq_bytes(sm) + kQOffW0;
    for (int warp = 0; warp < 6; ++warp) {
        const int t0 = 16 * (warp >> 1), n0 = 16 * (warp & 1);
        int32_t c[2][32][4] = {};
        for (int ks = 0; ks < 7; ++ks) {
            FragA8 a[32]; FragB8 b0[32], b1[32];
            for (int lane = 0; lane < 32; ++lane) {
                load_frag_a8(a8, kW0Pitch, 32 * ks, t0, lane, a[lane]);
                load_frag_b8(w0, kW0Pitch, 32 * ks, n0, lane, b0[lane]);
                load_frag_b8(w0, kW0Pitch, 32 * ks, n0 + 8, lane, b1[lane]);
            }
            warp_mma_s8(c[0], a, b0);
            warp_mma_s8(c[1], a, b1);
        }
        for (int lane = 0; lane < 32; ++lane) { nnq_fc_store_tile(sm, W, t0, n0, lane, c[0][lane]); nnq_fc_store_tile(sm, W, t0, n0 + 8, lane, c[1][lane]); }
    }
}

template <int L>
void emul_q_pointwise_mma(int32_t *sm, const NnWeightsI8 &W) {
    constexpr int cin = kGeom[L].cin;
    const int8_t *d8 = nnq_bytes(sm) + kQOffD8, *wt = nnq_bytes(sm) + kQOffPw + L * 64 * kPwPitch;
    for (int warp = 0; warp < kNnThreads / 32; ++warp) {
        const int t0 = 16 * (warp / 3), nt0 = 3 * (warp % 3), ntc = (warp % 3) == 2 ? 2 : 3;
        int32_t c[3][32][4] = {};
        for (int ks = 0; ks < cin / 32; ++ks) {
            FragA8 a[32];
            for (int lane = 0; lane < 32; ++lane) load_frag_a8(d8, kPwPitch, 32 * ks, t0, lane, a[lane]);
            for (int i = 0; i < ntc; ++i) {
                FragB8 b[32];
                for (int lane = 0; lane < 32; ++lane) load_frag_b8(wt, kPwPitch, 32 * ks, 8 * (nt0 + i), lane, b[lane]);
                warp_mma_s8(c[i], a, b);
            }
        }
        for (int i = 0; i < ntc; ++i)
            for (int lane = 0; lane < 32; ++lane) nnq_pw_store_tile<L>(sm, W, t0, 8 * (nt0 + i), lane, c[i][lane]);
    }
}
}  // namespace

namespace {
void unpack_i8_weights(const void *const *wp, const int32_t *zp12, const int32_t *head3, float in_scale, NnWeightsI8 &W, I8MmaOperands &ops);
}

extern "C" int emul_nn_i8(const void *const *wp /* see order below */, const int32_t *zp12, const int32_t *head3, float in_scale,
                          int8_t *state, int8_t *pend, int n_pend, const void *rows, int n_rows, int row_type,
                          int n_streams, float *probs, int max_probs) {
    NnWeightsI8 W;
    int k = 0;
    W.w0 = (const int8_t *)wp[k++]; W.b0 = (const int32_t *)wp[k++]; W.m0 = (const int32_t *)wp[k++]; W.s0 = (const int32_t *)wp[k++];
    for (int i = 0; i < 4; ++i) {
        W.dw_w[i] = (const int8_t *)wp[k++]; W.dw_b[i] = (const int32_t *)wp[k++]; W.dw_m[i] = (const int32_t *)wp[k++]; W.dw_s[i] = (const int32_t *)wp[k++];
        W.pw_w[i] = (const int8_t *)wp[k++]; W.pw_b[i] = (const int32_t *)wp[k++]; W.pw_m[i] = (const int32_t *)wp[k++]; W.pw_s[i] = (const int32_t *)wp[k++];
    }
    W.head_w = (const int8_t *)wp[k++]; W.lut = (const int8_t *)wp[k++];
    W.head_bias = head3[0]; W.head_mult = head3[1]; W.head_shift = head3[2];
    memcpy(W.zp, zp12, sizeof W.zp);
    W.in_scale = in_scale;
    I8MmaOperands ops;
    build_i8_mma_operands(W.w0, W.b0, W.pw_w, W.pw_b, W.zp, &ops);
    W.w0t = ops.w0t.data(); W.b0f = ops.b0f.data();
    if (getenv("MWW_NO_QLUT") == nullptr) {      // as mww_create does: uint16 features are quantised through the table
        build_feature_qlut(W.in_scale, W.zp[0], &ops.qlut);
        W.qlut = ops.qlut.data();
    }
    for (int i = 0; i < 4; ++i) { W.pwt[i] = ops.pwt[i].data(); W.pw_bf[i] = ops.pw_bf[i].data(); }
    const int n_virtual = n_pend + n_rows;
    const int n_steps = n_virtual / 3;
    const size_t row_bytes = (size_t)kNumChannels * (row_type == 1 ? 4 : (row_type == 0 ? 2 : 1));
    std::vector<int32_t> smv(kNnI8SmemBytes / 4 + 4);
    int32_t *sm = smv.data();
    for (int s = 0; s < n_streams; ++s) {
        for (auto &v : smv) v = 0x5A5A5A5A;
        int8_t *my_state = state + (size_t)s * kStateFloats;
        int8_t *my_pend = pend + (size_t)s * 2 * kNumChannels;
        NnInputI8 in;
        in.ring0 = my_state; in.pend = my_pend; in.n_pend = n_pend;
        in.rows = static_cast<const char *>(rows) + (size_t)s * n_rows * row_bytes;
        in.n_rows = n_rows; in.row_type = row_type;
#define ALL(stmt) for (int tid = 0; tid < kNnThreads; ++tid) { stmt; }
        ALL(nnq_load_state(tid, sm, my_state, W));
        ALL(nnq_load_weights(tid, sm, W));
        for (int step0 = 0; step0 < n_steps; step0 += kTT) {
            const int n = n_steps - step0 < kTT ? n_steps - step0 : kTT;
            ALL(nnq_load_features(tid, sm, in, W, step0, n));
            emul_q_first_conv_mma(sm, W);
            ALL(nnq_depthwise<0>(tid, sm, W)); emul_q_pointwise_mma<0>(sm, W);
            ALL(nnq_depthwise<1>(tid, sm, W)); emul_q_pointwise_mma<1>(sm, W);
            ALL(nnq_depthwise<2>(tid, sm, W)); emul_q_pointwise_mma<2>(sm, W);
            ALL(nnq_depthwise<3>(tid, sm, W)); emul_q_pointwise_mma<3>(sm, W);
            ALL(nnq_head_partial(tid, sm, W));
            ALL(nnq_head_finish(tid, sm, W, n, probs + (size_t)s * max_probs + step0));
            std::vector<float> tmp((size_t)kNnThreads * 5 * kShiftPerThread);
            ALL(nn_shift_read(tid, reinterpret_cast<const float *>(sm), n, *reinterpret_cast<float(*)[5][kShiftPerThread]>(&tmp[(size_t)tid * 5 * kShiftPerThread])));
            ALL(nn_shift_write(tid, reinterpret_cast<float *>(sm), *reinterpret_cast<float(*)[5][kShiftPerThread]>(&tmp[(size_t)tid * 5 * kShiftPerThread])));
        }
        std::vector<NnTailI8> tails(kNnThreads);
        ALL(nnq_tail_read(tid, in, W, n_steps, n_virtual, tails[tid]));
        ALL(nnq_tail_write(tid, sm, my_state, my_pend, W, tails[tid]));
#undef ALL
    }
    return n_steps;
}

extern "C" void emul_fill_state_i8(const int32_t *zp12, int8_t *state, int8_t *pend, int n_streams) {
    NnWeightsI8 W;
    memcpy(W.zp, zp12, sizeof W.zp);
    for (int s = 0; s < n_streams; ++s) {
        for (int e = 0; e < kStateFloats; ++e) state[(size_t)s * kStateFloats + e] = nnq_reset_value(W, e);
        for (int e = 0; e < 2 * kNumChannels; ++e) pend[(size_t)s * 2 * kNumChannels + e] = (int8_t)W.zp[0];
    }
}

extern "C" int32_t emul_mbqm(int32_t x, int32_t mult, int32_t shift) { return mbqm(x, mult, shift); }


// ---- live-step fp32 kernel (mww_nn_live.cuh) ---------------------------------------------------------------
namespace {
void emul_live_first_conv(float *sm, const float *w0, int w0_pitch) {
    for (int warp = 0; warp < kLiveThreads / 32; ++warp) {
        const int r0 = 16 * (warp >> 2), n0 = 8 * (warp & 3);
        float c[32][4] = {};
        for (int ks = 0; ks < 25; ++ks) {
            FragA a[32]; FragB b[32];
            for (int lane = 0; lane < 32; ++lane) { load_frag_b(w0, w0_pitch, 8 * ks, n0, lane, b[lane]); load_frag_a(sm + kLiveOffA, kLivePitch, 8 * ks, r0, lane, a[lane]); }
            warp_mma_3xtf32(c, a, b);
        }
        for (int lane = 0; lane < 32; ++lane) live_fc_store_tile(sm, r0, n0, lane, c[lane]);
    }
}
template <int L, bool SMEM_ALL = false>
void emul_live_pointwise(float *sm, const NnWeightsF32 &W) {
    constexpr int cin = kGeom[L].cin;
    for (int warp = 0; warp < kLiveThreads / 32; ++warp) {
        const int r0 = 16 * (warp >> 2), n0 = 16 * (warp & 3);
        float c[2][32][4] = {};
        for (int ks = 0; ks < cin / 8; ++ks) {
            FragA a[32]; FragB b0[32], b1[32];
            for (int lane = 0; lane < 32; ++lane) {
                load_frag_a(sm + kLiveOffD, kLivePitch, 8 * ks, r0, lane, a[lane]);
                const float *wsm = L == 0 ? (SMEM_ALL ? sm + kLive2OffPw0 : W.pw_w[0]) : sm + live_pw_offset<L>();
                const int wld = (L == 0 && !SMEM_ALL) ? 64 : kWLd;
                load_frag_b(wsm, wld, 8 * ks, n0, lane, b0[lane]);
                load_frag_b(wsm, wld, 8 * ks, n0 + 8, lane, b1[lane]);
            }
            warp_mma_3xtf32(c[0], a, b0);
            warp_mma_3xtf32(c[1], a, b1);
        }
        const float *bias = SMEM_ALL ? sm + kLive2OffSmall + kLive2SmallPwBias + 64 * L : W.pw_b[L];
        for (int lane = 0; lane < 32; ++lane) { live_pw_store_tile_b(sm, bias, r0, n0, lane, c[0][lane]); live_pw_store_tile_b(sm, bias, r0, n0 + 8, lane, c[1][lane]); }
    }
}
}  // namespace

extern "C" int emul_nn_f32_live(const float *const *wp, float *state, float *pend, int n_pend, const void *rows, int rows_are_f32,
                                int n_streams, float *probs, int probs_stride, const int *heads5) {
    NnWeightsF32 W;
    W.w0 = wp[0];
    for (int i = 0; i < 4; ++i) { W.dw_w[i] = wp[1 + i]; W.dw_b[i] = wp[5 + i]; W.pw_w[i] = wp[9 + i]; W.pw_b[i] = wp[13 + i]; }
    W.head_w = wp[17]; W.head_b = wp[18];
    LiveHeads heads;
    for (int i = 0; i < 5; ++i) heads.h[i] = heads5[i];
    LiveInput in;
    in.state = state; in.pend = pend; in.n_pend = n_pend; in.rows = rows;
    in.rows_stream_stride_bytes = 3 * kNumChannels * (rows_are_f32 ? 4 : 2); in.rows_are_f32 = rows_are_f32;
    std::vector<float> smv(kLiveSmemFloats, -777.f);
    float *sm = smv.data();
#define ALLL(stmt) for (int tid = 0; tid < kLiveThreads; ++tid) { stmt; }
    ALLL(live_load_weights(tid, sm, W));
    const int n_groups = (n_streams + kLiveStreams - 1) / kLiveStreams;
    for (int g = 0; g < n_groups; ++g) {
        const long long s0 = (long long)g * kLiveStreams;
        const int n_valid = n_streams - (int)s0 < kLiveStreams ? n_streams - (int)s0 : kLiveStreams;
        std::vector<float> keeps((size_t)kLiveThreads * 4 * kLiveKeep);
#define KP(tid) (*reinterpret_cast<float(*)[4][kLiveKeep]>(&keeps[(size_t)(tid) * 4 * kLiveKeep]))
        ALLL(live_build_a(tid, sm, in, s0, n_valid, KP(tid)));
        ALLL(live_write_tail(tid, state, pend, s0, n_valid, KP(tid)));
#undef KP
        emul_live_first_conv(sm, W.w0, 32);
        ALLL(live_depthwise<0>(tid, sm, W, state, s0, n_valid, heads.h[0])); emul_live_pointwise<0>(sm, W);
        ALLL(live_depthwise<1>(tid, sm, W, state, s0, n_valid, heads.h[1])); emul_live_pointwise<1>(sm, W);
        ALLL(live_depthwise<2>(tid, sm, W, state, s0, n_valid, heads.h[2])); emul_live_pointwise<2>(sm, W);
        ALLL(live_depthwise<3>(tid, sm, W, state, s0, n_valid, heads.h[3])); emul_live_pointwise<3>(sm, W);
        ALLL(live_head_partial(tid, sm, W, state, s0, n_valid, heads.h[4]));
        ALLL(live_head_finish(tid, sm, W, s0, n_valid, probs, probs_stride));
    }
#undef ALLL
    return 1;
}

// v2: the warp-specialised live kernel (nn_f32_live2_kernel).  Streamers (512 threads) fill P for a group, then the chain
// (256 threads) consumes it; on the GPU the streamers run up to two groups ahead -- the emulation runs them one group at a
// time, which is the order the named barriers enforce per buffer.  `order` 1 walks every phase's threads in descending order.
extern "C" int emul_nn_f32_live2(const float *const *wp, float *state, float *pend, int n_pend, const void *rows, int rows_are_f32,
                                 int n_streams, float *probs, int probs_stride, const int *heads5, int order) {
    NnWeightsF32 W;
    W.w0 = wp[0];
    for (int i = 0; i < 4; ++i) { W.dw_w[i] = wp[1 + i]; W.dw_b[i] = wp[5 + i]; W.pw_w[i] = wp[9 + i]; W.pw_b[i] = wp[13 + i]; }
    W.head_w = wp[17]; W.head_b = wp[18];
    LiveHeads heads;
    for (int i = 0; i < 5; ++i) heads.h[i] = heads5[i];
    LiveInput in;
    in.state = state; in.pend = pend; in.n_pend = n_pend; in.rows = rows;
    in.rows_stream_stride_bytes = 3 * kNumChannels * (rows_are_f32 ? 4 : 2); in.rows_are_f32 = rows_are_f32;
    std::vector<float> smv(kLive2SmemFloats, -777.f);
    float *sm = smv.data();
#define CHAIN(stmt) for (int i_ = 0; i_ < kLive2ChainThreads; ++i_) { const int tid = order ? kLive2ChainThreads - 1 - i_ : i_; stmt; }
#define STREAM(stmt) for (int i_ = 0; i_ < kLive2StreamThreads; ++i_) { const int st = order ? kLive2StreamThreads - 1 - i_ : i_; stmt; }
    for (int tid = 0; tid < kLive2Threads; ++tid)
        for (int L = 1; L < 4; ++L) {
            float *dst = sm + (L == 1 ? kLiveOffPw1 : (L == 2 ? kLiveOffPw2 : kLiveOffPw3));
            for (int e = tid; e < 64 * 64; e += kLive2Threads) dst[(e >> 6) * kWLd + (e & 63)] = W.pw_w[L][e];
        }
    for (int tid = 0; tid < kLive2Threads; ++tid) live2_stage_chain_tables(tid, kLive2Threads, sm, W);
    const int n_groups = (n_streams + kLiveStreams - 1) / kLiveStreams;
    for (int g = 0; g < n_groups; ++g) {
        const long long s0 = (long long)g * kLiveStreams;
        const int n_valid = n_streams - (int)s0 < kLiveStreams ? n_streams - (int)s0 : kLiveStreams;
        float *p_buf = sm + kLive2OffP + (g & 1) * kLive2PFloats;
        STREAM(live2_stream_group(st, W, state, s0, n_valid, heads, p_buf));
        STREAM(live2_build_a<kLive2StreamThreads>(st, sm, in, s0, n_valid));
        emul_live_first_conv(sm, sm + kLive2OffW0, kLive2W0Pitch);
        CHAIN(live2_write_tail(tid, sm, in, state, pend, s0, n_valid));
        CHAIN(live2_dw_from_p<0>(tid, sm, state, s0, n_valid, heads.h[0], p_buf)); emul_live_pointwise<0, true>(sm, W);
        CHAIN(live2_dw_from_p<1>(tid, sm, state, s0, n_valid, heads.h[1], p_buf)); emul_live_pointwise<1, true>(sm, W);
        CHAIN(live2_dw_from_p<2>(tid, sm, state, s0, n_valid, heads.h[2], p_buf)); emul_live_pointwise<2, true>(sm, W);
        CHAIN(live2_dw_from_p<3>(tid, sm, state, s0, n_valid, heads.h[3], p_buf)); emul_live_pointwise<3, true>(sm, W);
        CHAIN(live2_dw_from_p<4>(tid, sm, state, s0, n_valid, heads.h[4], p_buf));
        CHAIN(live_head_finish_b(tid, sm, sm[kLive2OffSmall + kLive2SmallHeadBias], s0, n_valid, probs, probs_stride));
    }
#undef CHAIN
#undef STREAM
    return 1;
}

// v3: the bulk-copy kernel (nn_f32_live3_kernel).  On the GPU a producer thread copies each stream's rings 1..5 into a shared
// memory stage and nine "P" warps (one ring column per thread) reduce it; six window warps build the first-conv window (and move
// the pending rows) a group ahead; the chain is v2's with the first conv's weights read from global memory.  The emulation runs
// the same phase functions with the stage = the stream's state in place (a short last group re-reads its last valid stream, as
// the producer does), window loads of a group before its chain.
template <int I>
static void emul_live3_p(const NnWeightsF32 &W, const float *state, long long s0, int n_valid, int head, float *sm, int order) {
    constexpr int C = live_ring_cols(I);
    for (int i_ = 0; i_ < C; ++i_) {
        const int c = order ? C - 1 - i_ : i_;
        float w[live_ring_rows(I)], bias;
        live3_p_taps<I>(W, c, head, w, bias);
        float *p_col = sm + kLive2OffP + (live2_col_base(I) + c) * kLive2PPitch;
        for (int sl = 0; sl < kLiveStreams; ++sl) {
            const long long stream = s0 + (sl < n_valid ? sl : n_valid - 1);
            p_col[sl] = live3_p_sum<I>(state + (size_t)stream * kStateFloats + kStateOff[1], c, w, bias);
        }
    }
}
extern "C" int emul_nn_f32_live3(const float *const *wp, float *state, float *pend, int n_pend, const void *rows, int rows_are_f32,
                                 int n_streams, float *probs, int probs_stride, const int *heads5, int order) {
    NnWeightsF32 W;
    W.w0 = wp[0];
    for (int i = 0; i < 4; ++i) { W.dw_w[i] = wp[1 + i]; W.dw_b[i] = wp[5 + i]; W.pw_w[i] = wp[9 + i]; W.pw_b[i] = wp[13 + i]; }
    W.head_w = wp[17]; W.head_b = wp[18];
    LiveHeads heads;
    for (int i = 0; i < 5; ++i) heads.h[i] = heads5[i];
    LiveInput in;
    in.state = state; in.pend = pend; in.n_pend = n_pend; in.rows = rows;
    in.rows_stream_stride_bytes = 3 * kNumChannels * (rows_are_f32 ? 4 : 2); in.rows_are_f32 = rows_are_f32;
    std::vector<float> smv(kLive2SmemFloats, -777.f);
    float *sm = smv.data();
#define CHAIN(stmt) for (int i_ = 0; i_ < kLive2ChainThreads; ++i_) { const int tid = order ? kLive2ChainThreads - 1 - i_ : i_; stmt; }
#define WINDOW(stmt) for (int i_ = 0; i_ < kLive3WindowThreads; ++i_) { const int at = order ? kLive3WindowThreads - 1 - i_ : i_; stmt; }
    for (int tid = 0; tid < kLive2Threads; ++tid)
        for (int L = 1; L < 4; ++L) {
            float *dst = sm + (L == 1 ? kLiveOffPw1 : (L == 2 ? kLiveOffPw2 : kLiveOffPw3));
            for (int e = tid; e < 64 * 64; e += kLive2Threads) dst[(e >> 6) * kWLd + (e & 63)] = W.pw_w[L][e];
        }
    for (int tid = 0; tid < kLive2Threads; ++tid) live2_stage_chain_tables(tid, kLive2Threads, sm, W, false);
    const int n_groups = (n_streams + kLiveStreams - 1) / kLiveStreams;
    std::vector<float> vals((size_t)kLive3WindowThreads * kLive3WindowPerThread);
    for (int g = 0; g < n_groups; ++g) {
        const long long s0 = (long long)g * kLiveStreams;
        const int n_valid = n_streams - (int)s0 < kLiveStreams ? n_streams - (int)s0 : kLiveStreams;
        emul_live3_p<0>(W, state, s0, n_valid, heads.h[0], sm, order);
        emul_live3_p<1>(W, state, s0, n_valid, heads.h[1], sm, order);
        emul_live3_p<2>(W, state, s0, n_valid, heads.h[2], sm, order);
        emul_live3_p<3>(W, state, s0, n_valid, heads.h[3], sm, order);
        emul_live3_p<4>(W, state, s0, n_valid, heads.h[4], sm, order);
        // window warps: every load of the group (old pending rows included) precedes the pending-row stores (named barrier)
        WINDOW({ float (&v)[kLive3WindowPerThread] = *reinterpret_cast<float (*)[kLive3WindowPerThread]>(&vals[(size_t)at * kLive3WindowPerThread]);
                 live3_window_load(at, in, s0, n_valid, v); });
        if (n_pend != 0) WINDOW(live3_pend_store(at, in, pend, s0, n_valid));
        WINDOW({ const float (&v)[kLive3WindowPerThread] = *reinterpret_cast<const float (*)[kLive3WindowPerThread]>(&vals[(size_t)at * kLive3WindowPerThread]);
                 live3_window_store(at, sm, v); });
        const float *p_buf = sm + kLive2OffP;
        emul_live_first_conv(sm, W.w0, 32);
        CHAIN(live3_write_ring0(tid, sm, state, s0, n_valid));
        CHAIN(live2_dw_from_p<0>(tid, sm, state, s0, n_valid, heads.h[0], p_buf)); emul_live_pointwise<0, true>(sm, W);
        CHAIN(live2_dw_from_p<1>(tid, sm, state, s0, n_valid, heads.h[1], p_buf)); emul_live_pointwise<1, true>(sm, W);
        CHAIN(live2_dw_from_p<2>(tid, sm, state, s0, n_valid, heads.h[2], p_buf)); emul_live_pointwise<2, true>(sm, W);
        CHAIN(live2_dw_from_p<3>(tid, sm, state, s0, n_valid, heads.h[3], p_buf)); emul_live_pointwise<3, true>(sm, W);
        CHAIN(live2_dw_from_p<4>(tid, sm, state, s0, n_valid, heads.h[4], p_buf));
        CHAIN(live_head_finish_b(tid, sm, sm[kLive2OffSmall + kLive2SmallHeadBias], s0, n_valid, probs, probs_stride));
    }
#undef CHAIN
#undef WINDOW
    return 1;
}

extern "C" void emul_nn_live_canonicalise(float *state, int n_streams, const int *heads5) {
    LiveHeads heads;
    for (int i = 0; i < 5; ++i) heads.h[i] = heads5[i];
    for (long long s = 0; s < n_streams; ++s)
        for (int col = 0; col < 288; ++col) live_canonicalise_column(state, s, col, heads);
}


extern "C" void emul_feature_qlut(float in_scale, int zp_in, int8_t *out65536) {
    std::vector<int8_t> t;
    build_feature_qlut(in_scale, zp_in, &t);
    memcpy(out65536, t.data(), t.size());
}

// ---- wgmma clip kernel: operand layout (mww_nn_tc_prep.h) ------------------------------------------------------
#include "../../microwakeword_b200/csrc/mww_nn_tc_prep.h"
extern "C" unsigned emul_sw128_off(int row, int kk) { return sw128_off(row, kk); }
// lays [K][N] weights out like mww_create does; returns the byte count (out may be NULL to query it)
extern "C" long long emul_tc_layout(const float *w, int K, int N, unsigned char *out, long long cap) {
    std::vector<unsigned char> blob;
    tc_layout(w, K, N, &blob);
    if (out && (long long)blob.size() <= cap) memcpy(out, blob.data(), blob.size());
    return (long long)blob.size();
}

// ---- live-step int8 kernel (mww_nn_i8_live.cuh) -------------------------------------------------------------
#include "../../microwakeword_b200/csrc/mww_nn_i8_live.cuh"
namespace {
void unpack_i8_weights(const void *const *wp, const int32_t *zp12, const int32_t *head3, float in_scale, NnWeightsI8 &W, I8MmaOperands &ops) {
    int k = 0;
    W.w0 = (const int8_t *)wp[k++]; W.b0 = (const int32_t *)wp[k++]; W.m0 = (const int32_t *)wp[k++]; W.s0 = (const int32_t *)wp[k++];
    for (int i = 0; i < 4; ++i) {
        W.dw_w[i] = (const int8_t *)wp[k++]; W.dw_b[i] = (const int32_t *)wp[k++]; W.dw_m[i] = (const int32_t *)wp[k++]; W.dw_s[i] = (const int32_t *)wp[k++];
        W.pw_w[i] = (const int8_t *)wp[k++]; W.pw_b[i] = (const int32_t *)wp[k++]; W.pw_m[i] = (const int32_t *)wp[k++]; W.pw_s[i] = (const int32_t *)wp[k++];
    }
    W.head_w = (const int8_t *)wp[k++]; W.lut = (const int8_t *)wp[k++];
    W.head_bias = head3[0]; W.head_mult = head3[1]; W.head_shift = head3[2];
    memcpy(W.zp, zp12, sizeof W.zp);
    W.in_scale = in_scale;
    build_i8_mma_operands(W.w0, W.b0, W.pw_w, W.pw_b, W.zp, &ops);
    W.w0t = ops.w0t.data(); W.b0f = ops.b0f.data();
    if (getenv("MWW_NO_QLUT") == nullptr) {      // as mww_create does: uint16 features are quantised through the table
        build_feature_qlut(W.in_scale, W.zp[0], &ops.qlut);
        W.qlut = ops.qlut.data();
    }
    for (int i = 0; i < 4; ++i) { W.pwt[i] = ops.pwt[i].data(); W.pw_bf[i] = ops.pw_bf[i].data(); }
}

void emul_livq_first_conv(uint8_t *smb, const NnWeightsI8 &W) {
    const int8_t *a8 = reinterpret_cast<const int8_t *>(smb + kLqOffA), *w0 = reinterpret_cast<const int8_t *>(smb + kLqOffW0);
    for (int warp = 0; warp < 8; ++warp) {
        const int r0 = 16 * (warp >> 2), n0 = 8 * (warp & 3);
        int32_t c[32][4] = {};
        for (int ks = 0; ks < 7; ++ks) {
            FragA8 a[32]; FragB8 b[32];
            for (int lane = 0; lane < 32; ++lane) { load_frag_a8(a8, kW0Pitch, 32 * ks, r0, lane, a[lane]); load_frag_b8(w0, kW0Pitch, 32 * ks, n0, lane, b[lane]); }
            warp_mma_s8(c, a, b);
        }
        for (int lane = 0; lane < 32; ++lane) livq_fc_store_tile(smb, W, r0, n0, lane, c[lane]);
    }
}
template <int L>
void emul_livq_pointwise(uint8_t *smb, const NnWeightsI8 &W) {
    constexpr int cin = kGeom[L].cin;
    const int8_t *d8 = reinterpret_cast<const int8_t *>(smb + kLqOffD), *wt = reinterpret_cast<const int8_t *>(smb + kLqOffPw + L * 64 * kPwPitch);
    for (int warp = 0; warp < 8; ++warp) {
        const int r0 = 16 * (warp >> 2), n0 = 16 * (warp & 3);
        int32_t c[2][32][4] = {};
        for (int ks = 0; ks < cin / 32; ++ks) {
            FragA8 a[32]; FragB8 b0[32], b1[32];
            for (int lane = 0; lane < 32; ++lane) {
                load_frag_a8(d8, kPwPitch, 32 * ks, r0, lane, a[lane]);
                load_frag_b8(wt, kPwPitch, 32 * ks, n0, lane, b0[lane]);
                load_frag_b8(wt, kPwPitch, 32 * ks, n0 + 8, lane, b1[lane]);
            }
            warp_mma_s8(c[0], a, b0);
            warp_mma_s8(c[1], a, b1);
        }
        for (int lane = 0; lane < 32; ++lane) { livq_pw_store_tile<L>(smb, W, r0, n0, lane, c[0][lane]); livq_pw_store_tile<L>(smb, W, r0, n0 + 8, lane, c[1][lane]); }
    }
}
}  // namespace

extern "C" int emul_nn_i8_live(const void *const *wp, const int32_t *zp12, const int32_t *head3, float in_scale, int8_t *state, int8_t *pend,
                               int n_pend, const void *rows, int row_type, int n_streams, float *probs, int probs_stride, const int *heads5) {
    NnWeightsI8 W;
    I8MmaOperands ops;
    unpack_i8_weights(wp, zp12, head3, in_scale, W, ops);
    LiveHeads heads;
    for (int i = 0; i < 5; ++i) heads.h[i] = heads5[i];
    LiveInputI8 in;
    in.state = state; in.pend = pend; in.n_pend = n_pend; in.rows = rows;
    in.rows_stream_stride_bytes = 3 * kNumChannels * (row_type == 1 ? 4 : (row_type == 0 ? 2 : 1)); in.row_type = row_type;
    std::vector<uint8_t> smv(kLiveQSmemBytes + 16, 0xA5);
    uint8_t *smb = smv.data();
    smb += (16 - reinterpret_cast<uintptr_t>(smb) % 16) % 16;
#define ALLQ(stmt) for (int tid = 0; tid < kLiveQThreads; ++tid) { stmt; }
    ALLQ(livq_load_weights(tid, smb, W));
    const int n_groups = (n_streams + kLiveStreams - 1) / kLiveStreams;
    for (int g = 0; g < n_groups; ++g) {
        const long long s0 = (long long)g * kLiveStreams;
        const int n_valid = n_streams - (int)s0 < kLiveStreams ? n_streams - (int)s0 : kLiveStreams;
        std::vector<uint32_t> keeps((size_t)kLiveQThreads * 4 * kLqKeep);
#define KQ(tid) (*reinterpret_cast<uint32_t(*)[4][kLqKeep]>(&keeps[(size_t)(tid) * 4 * kLqKeep]))
        ALLQ(livq_build_a(tid, smb, in, W, s0, n_valid, KQ(tid)));
        ALLQ(livq_write_tail(tid, state, pend, s0, n_valid, KQ(tid)));
#undef KQ
        emul_livq_first_conv(smb, W);
        ALLQ(livq_depthwise<0>(tid, smb, W, state, s0, n_valid, heads.h[0])); emul_livq_pointwise<0>(smb, W);
        ALLQ(livq_depthwise<1>(tid, smb, W, state, s0, n_valid, heads.h[1])); emul_livq_pointwise<1>(smb, W);
        ALLQ(livq_depthwise<2>(tid, smb, W, state, s0, n_valid, heads.h[2])); emul_livq_pointwise<2>(smb, W);
        ALLQ(livq_depthwise<3>(tid, smb, W, state, s0, n_valid, heads.h[3])); emul_livq_pointwise<3>(smb, W);
        ALLQ(livq_head_partial(tid, smb, W, state, s0, n_valid, heads.h[4]));
        ALLQ(livq_head_finish(tid, smb, W, s0, n_valid, probs, probs_stride));
    }
#undef ALLQ
    return 1;
}

extern "C" void emul_nn_i8_live_canonicalise(int8_t *state, int n_streams, const int *heads5) {
    LiveHeads heads;
    for (int i = 0; i < 5; ++i) heads.h[i] = heads5[i];
    for (long long s = 0; s < n_streams; ++s)
        for (int col = 0; col < 288; ++col) livq_canonicalise_column(state, s, col, heads);
}
