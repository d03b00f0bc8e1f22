// tests/host_emul/emul_hybrid.cc -- TEST INFRASTRUCTURE: CPU execution of the hybrid (fp32 graph, int8-weight ops) phase
// functions of microwakeword_b200/csrc/mww_nn_generic.cuh in exactly the order nn_generic_hybrid_kernel issues them, every
// barrier a phase boundary, shared memory poisoned before each stream.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../microwakeword_b200/csrc/mww_nn_generic.cuh"

using namespace mww;

// threads of a phase run one after the other, in ascending or descending order (the order must not matter)
static int g_reverse = 0;
extern "C" void emul_hy_thread_order(int reversed) { g_reverse = reversed; }
#define HY_ALL(...) for (int t_ = 0; t_ < kGenThreads; ++t_) { const int tid = g_reverse ? kGenThreads - 1 - t_ : t_; __VA_ARGS__; }

// the device quantiser on one tensor: per-thread min / max partials, gen_hy_qparams, hy_code (the known-answer tests)
extern "C" void emul_hy_quantize(int mode, const float *x, int n, int8_t *q, float *scale, int32_t *zp) {
    GenHybrid H = GenHybrid();
    H.sm_par = 0; H.sm_red = 4 * kHyMaxQ; H.sm_q = H.sm_red + 2 * kHyMaxQ * kGenThreads; H.sm_elems = H.sm_q;
    std::vector<float> smv(H.sm_elems, -1234.5f);
    float *sm = smv.data();
    HY_ALL({
        float mn = INFINITY, mx = -INFINITY;
        for (int i = tid; i < n; i += kGenThreads) { mn = x[i] < mn ? x[i] : mn; mx = x[i] > mx ? x[i] : mx; }
        hy_put_partial(sm, H, 0, tid, mn, mx);
    });
    HY_ALL(gen_hy_qparams(tid, sm, H, tid == 0 ? mode : kHyFloat));
    for (int i = 0; i < n; ++i) q[i] = (int8_t)hy_code(sm + H.sm_par, mode, x[i]);
    *scale = sm[H.sm_par];
    *zp = (int32_t)sm[H.sm_par + 2];
}

// wf: w0, per block {dw_w, dw_b, pw_w, pw_b}, head_w, head_b (fp32 container tensors)
// wh: hy/first_conv/{w,scale}, per block hy/b{i}/dw/{w,scale}, hy/b{i}/pw/{w,scale}, hy/head/{w,scale}; NULL where absent
extern "C" int emul_hy_run(const int32_t *arch, int n_arch, const int32_t *modes, int n_modes, const float *const *wf, const void *const *wh,
                           float *state, float *pend, int n_pend, const void *rows, int n_rows, int row_type, int n_streams,
                           float *probs, int max_probs, long long *sm_bytes_out) {
    GenArch A;
    if (gen_arch_from_tensor(arch, n_arch, &A)) return -1;
    GenHybrid H = GenHybrid();
    if (gen_hybrid_layout(A, arch, modes, n_modes, &H)) return -3;
    if (sm_bytes_out) *sm_bytes_out = (long long)H.sm_elems * 4;
    GenWeightsF32 W = GenWeightsF32();
    int k = 0;
    W.w0 = wf[k++];
    for (int b = 0; b < A.n_blocks; ++b) { W.dw_w[b] = wf[k++]; W.dw_b[b] = wf[k++]; W.pw_w[b] = wf[k++]; W.pw_b[b] = wf[k++]; }
    W.head_w = wf[k++]; W.head_b = wf[k++];
    k = 0;
    H.w0 = (const int8_t *)wh[k++]; H.s0 = (const float *)wh[k++];
    for (int b = 0; b < A.n_blocks; ++b) {
        H.dw_w[b] = (const int8_t *)wh[k++]; H.dw_s[b] = (const float *)wh[k++];
        H.pw_w[b] = (const int8_t *)wh[k++]; H.pw_s[b] = (const float *)wh[k++];
    }
    H.head_w = (const int8_t *)wh[k++]; H.head_s = (const float *)wh[k++];
    const int n_steps = (n_pend + n_rows) / A.stride;
    if (n_steps > max_probs) return -2;
    const size_t row_bytes = (size_t)kNumChannels * (row_type == 1 ? 4 : 2);
    std::vector<float> smv(H.sm_elems);
    float *sm = smv.data();
    for (int s = 0; s < n_streams; ++s) {
        for (auto &v : smv) v = -1234.5f;   // poison
        float *my_state = state + (size_t)s * A.state_elems;
        float *my_pend = pend + (size_t)s * A.pend_cap * kNumChannels;
        GenInput<float> in;
        in.state = my_state; in.pend = my_pend; in.n_pend = n_pend;
        in.rows = static_cast<const char *>(rows) + (size_t)s * n_rows * row_bytes;
        in.n_rows = n_rows; in.row_type = row_type;
        HY_ALL(gen_f32_load_state(tid, sm, A, my_state));
        for (int t = 0; t < n_steps; ++t) {
            if (H.mode0 != kHyFloat) {
                HY_ALL(gen_hy_window(tid, sm, A, H, in, t));
                HY_ALL(gen_hy_qparams(tid, sm, H, tid == 0 ? H.mode0 : kHyFloat));
                HY_ALL(gen_hy_quant_window(tid, sm, A, H));
                HY_ALL(gen_hy_first_conv(tid, sm, A, H));
            } else {
                HY_ALL(gen_f32_window(tid, sm, A, in, t));
                HY_ALL(gen_f32_first_conv(tid, sm, A, W));
            }
            for (int b = 0; b < A.n_blocks; ++b) {
                const int pos = t % A.kmax[b];
                if (H.any_dw[b]) {
                    HY_ALL(gen_hy_block_insert(tid, sm, A, H, b, pos));
                    HY_ALL(gen_hy_qparams(tid, sm, H, tid < H.n_groups[b] ? H.g_mode[b][tid & (kHyMaxQ - 1)] : kHyFloat));
                    HY_ALL(gen_hy_quant_block(tid, sm, A, H, b, pos));
                    HY_ALL(gen_hy_depthwise(tid, sm, A, W, H, b, pos));
                } else {
                    HY_ALL(gen_f32_depthwise(tid, sm, A, W, b, pos));
                }
                if (H.mode_pw[b] != kHyFloat) {
                    HY_ALL(gen_hy_minmax_d(tid, sm, A, H, b));
                    HY_ALL(gen_hy_qparams(tid, sm, H, tid == 0 ? H.mode_pw[b] : kHyFloat));
                    HY_ALL(gen_hy_quant_d(tid, sm, A, H, b));
                    HY_ALL(gen_hy_pointwise(tid, sm, A, W, H, b));
                } else {
                    HY_ALL(gen_f32_pointwise(tid, sm, A, W, b));
                }
            }
            const int hpos = t % A.head_rows;
            if (H.mode_head != kHyFloat) {
                HY_ALL(gen_hy_head_insert(tid, sm, A, H, hpos));
                HY_ALL(gen_hy_qparams(tid, sm, H, tid == 0 ? H.mode_head : kHyFloat));
                HY_ALL(gen_hy_quant_head(tid, sm, A, H));
                HY_ALL(gen_hy_head_partial(tid, sm, A, H, hpos));
                HY_ALL(gen_hy_head_finish(tid, sm, A, W, H, probs + (size_t)s * max_probs + t));
            } else {
                HY_ALL(gen_f32_head_partial(tid, sm, A, W, hpos));
                HY_ALL(gen_f32_head_finish(tid, sm, A, W, probs + (size_t)s * max_probs + t));
            }
        }
        HY_ALL(gen_f32_tail_gather(tid, sm, A, in, n_steps));
        HY_ALL(gen_hy_tail_store(tid, sm, A, my_state, my_pend, A.ring0 + n_pend + n_rows - A.stride * n_steps, n_steps));
    }
    return n_steps;
}
