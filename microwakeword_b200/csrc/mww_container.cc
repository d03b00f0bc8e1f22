// mww_container.cc -- model container parsing (mww_container.h).  Tensor names and layouts: microwakeword_b200/model_file.py,
// the same names the CPU checker reads.
#include "mww_container.h"

#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/mww.h"
#include "mww_nn_i8_prep.h"

namespace mww {

namespace {

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

constexpr uint32_t kF32 = 0, kI8 = 1, kI32 = 2;     // container dtype codes

// the tensor-core kernels are compiled for the okay_nabu MixedNet (first conv 32x5 stride 3; MixConv [5],[7,11],[9,15],[23];
// pointwise 64x4; 17-row head)
const int32_t kOkayNabuArch[30] = {32, 5, 3, 40, 4, 17, 64, 1, 5, 0, 0, 0, 64, 2, 7, 11, 0, 0, 64, 2, 9, 15, 0, 0, 64, 1, 23, 0, 0, 0};

struct Reader {
    const uint8_t *blob; size_t n; ModelWeights *m; std::string *err;

    int fail(int code, const std::string &msg) { *err = msg; return code; }
    // appends `bytes` to the arena at the next 256-byte boundary; *field holds the offset until rebase()
    template <typename T>
    void put(const void *src, size_t bytes, const T **field) {
        const size_t off = (m->arena.size() + 255) / 256 * 256;
        m->arena.resize(off + bytes);
        memcpy(m->arena.data() + off, src, bytes);
        *field = reinterpret_cast<const T *>(off);
        m->fixups.push_back((size_t)(reinterpret_cast<const unsigned char *>(field) - reinterpret_cast<const unsigned char *>(m)));
    }
    // a tensor of `count` elements of `dtype`, copied into the arena
    template <typename T>
    int get(const char *name, uint32_t dtype, size_t count, const T **field) {
        static const size_t esz[6] = {4, 1, 4, 1, 2, 2};
        Tensor t;
        if (!find_tensor(blob, n, name, &t)) return fail(MWW_EMODEL, std::string("model container: missing tensor ") + name);
        if (t.dtype != dtype || t.nbytes != count * esz[dtype]) return fail(MWW_EMODEL, std::string("model container: wrong dtype/size for ") + name);
        put(t.data, (size_t)t.nbytes, field);
        return MWW_OK;
    }
    int scalar(const char *name, int32_t *out) {
        Tensor t;
        if (!find_tensor(blob, n, name, &t) || t.nbytes != 4) return fail(MWW_EMODEL, std::string("model container: ") + name);
        memcpy(out, t.data, 4);
        return MWW_OK;
    }
    // the arena's copy of a tensor get() placed (valid until the next put)
    template <typename T>
    const T *host(const T *field) const { return reinterpret_cast<const T *>(m->arena.data() + reinterpret_cast<uintptr_t>(field)); }
};

}  // namespace

const GenArch &okay_nabu_arch() {
    static const GenArch g = [] {
        GenArch a{};
        gen_arch_from_tensor(kOkayNabuArch, 30, &a);
        return a;
    }();
    return g;
}

void ModelWeights::rebase(const void *base) {
    for (size_t f : fixups) {
        unsigned char *slot = reinterpret_cast<unsigned char *>(this) + f;
        uintptr_t off;
        memcpy(&off, slot, sizeof off);
        const unsigned char *p = static_cast<const unsigned char *>(base) + off;
        memcpy(slot, &p, sizeof p);
    }
    std::vector<size_t>().swap(fixups);
    std::vector<unsigned char>().swap(arena);
    if (kind == ModelKind::kCompiledF32) {
        W.w0 = GW.w0; W.head_w = GW.head_w; W.head_b = GW.head_b;
        for (int i = 0; i < 4; ++i) { W.dw_w[i] = GW.dw_w[i]; W.dw_b[i] = GW.dw_b[i]; W.pw_w[i] = GW.pw_w[i]; W.pw_b[i] = GW.pw_b[i]; }
    } else if (kind == ModelKind::kCompiledI8) {
        Wq.w0 = GQ.w0; Wq.b0 = GQ.b0; Wq.m0 = GQ.m0; Wq.s0 = GQ.s0;
        for (int i = 0; i < 4; ++i) {
            Wq.dw_w[i] = GQ.dw_w[i]; Wq.dw_b[i] = GQ.dw_b[i]; Wq.dw_m[i] = GQ.dw_m[i]; Wq.dw_s[i] = GQ.dw_s[i];
            Wq.pw_w[i] = GQ.pw_w[i]; Wq.pw_b[i] = GQ.pw_b[i]; Wq.pw_m[i] = GQ.pw_m[i]; Wq.pw_s[i] = GQ.pw_s[i];
        }
        Wq.head_w = GQ.head_w; Wq.lut = GQ.lut;
        Wq.head_bias = GQ.head_bias; Wq.head_mult = GQ.head_mult; Wq.head_shift = GQ.head_shift;
        memcpy(Wq.zp, GQ.zp, sizeof Wq.zp);
        Wq.in_scale = GQ.in_scale;
    }
}

int parse_container(const uint8_t *blob, size_t n, ModelWeights *out, std::string *err) {
    Reader r{blob, n, out, err};
    ModelWeights &m = *out;
    Tensor arch;
    if (!find_tensor(blob, n, "arch", &arch) || arch.dtype != kI32) return r.fail(MWW_EMODEL, "model container: missing 'arch' tensor or bad magic/version");
    std::vector<int32_t> a(arch.nbytes / 4);
    if (!a.empty()) memcpy(a.data(), arch.data, a.size() * 4);
    GenArch &G = m.G;
    const int rc_arch = gen_arch_from_tensor(a.data(), (int)a.size(), &G);
    if (rc_arch == -1) return r.fail(MWW_EMODEL, "model container: malformed 'arch' tensor");
    if (rc_arch != 0 || (size_t)G.sm_elems * 4 > 200 * 1024)
        return r.fail(MWW_EUNSUPPORTED, "model container: architecture outside the supported range (first_conv_kernel_size >= stride, <= 8 blocks, "
                                        "<= 512 channels, kernels <= 64 taps, ring buffers of one stream within 200 KB)");
    // okay_nabu runs on the compiled kernels unless MWW_FORCE_GENERIC is set (tests compare the two paths).  A hybrid container of any
    // architecture, okay_nabu's included, runs on the generic hybrid kernel: the compiled fp32 kernels' arithmetic is not TFLite's
    // hybrid arithmetic.
    Tensor mode, probe;
    const bool has_mode = find_tensor(blob, n, "hy/mode", &mode), quantized = find_tensor(blob, n, "q/scales", &probe);
    const bool compiled = !has_mode && arch.nbytes == sizeof kOkayNabuArch && memcmp(arch.data, kOkayNabuArch, sizeof kOkayNabuArch) == 0 &&
                          getenv("MWW_FORCE_GENERIC") == nullptr;
    m.kind = compiled ? (quantized ? ModelKind::kCompiledI8 : ModelKind::kCompiledF32)
                      : (quantized ? ModelKind::kGenericI8 : (has_mode ? ModelKind::kHybrid : ModelKind::kGenericF32));
    const size_t k0f = (size_t)G.k0 * kNumChannels * G.c0;
    char name[64];
    int rc;
    if (!quantized) {
        GenWeightsF32 &W = m.GW;
        if ((rc = r.get("first_conv/w", kF32, k0f, &W.w0))) return rc;
        for (int i = 0; i < G.n_blocks; ++i) {
            snprintf(name, sizeof name, "b%d/dw/w", i); if ((rc = r.get(name, kF32, (size_t)G.kmax[i] * G.cin[i], &W.dw_w[i]))) return rc;
            snprintf(name, sizeof name, "b%d/dw/b", i); if ((rc = r.get(name, kF32, G.cin[i], &W.dw_b[i]))) return rc;
            snprintf(name, sizeof name, "b%d/pw/w", i); if ((rc = r.get(name, kF32, (size_t)G.cin[i] * G.cout[i], &W.pw_w[i]))) return rc;
            snprintf(name, sizeof name, "b%d/pw/b", i); if ((rc = r.get(name, kF32, G.cout[i], &W.pw_b[i]))) return rc;
        }
        if ((rc = r.get("head/w", kF32, (size_t)G.head_rows * G.c_last, &W.head_w))) return rc;
        if ((rc = r.get("head/b", kF32, 1, &W.head_b))) return rc;
        if (compiled) {
            // tensor-core operands, once per model (mww_nn_tc_prep.h): 3xTF32 split + slot layout, and the first conv's fp16
            // operands where its weights admit them
            const TcF16Scales sc = tc_f16_scales(r.host(W.w0));
            m.tc_f16 = sc.ok && getenv("MWW_TC_TF32") == nullptr;
            std::vector<unsigned char> fc, pw[4], fc16;
            tc_layout(r.host(W.w0), G.k0 * kNumChannels, G.c0, &fc);
            for (int i = 0; i < 4; ++i) tc_layout(r.host(W.pw_w[i]), G.cin[i], G.cout[i], &pw[i]);
            if (m.tc_f16) tc_layout_f16(r.host(W.w0), G.k0 * kNumChannels, G.c0, kFeatureScale, sc.s_fc, &fc16);
            r.put(fc.data(), fc.size(), &m.TW.fc);
            for (int i = 0; i < 4; ++i) r.put(pw[i].data(), pw[i].size(), &m.TW.pw[i]);
            if (m.tc_f16) {
                r.put(fc16.data(), fc16.size(), &m.TW.fc16);
                m.TW.fc_out = ldexpf(1.f, -sc.s_fc);
            }
        }
        if (!has_mode) return MWW_OK;
        // hybrid layers (model_file.py): int8 weights + per-channel scales next to the fp32 tensors
        GenHybrid &H = m.GH;
        if (mode.dtype != kI32 || mode.nbytes % 4 != 0 || mode.nbytes > 4 * (2 + 5 * kGenMaxBlocks)) return r.fail(MWW_EMODEL, "model container: malformed 'hy/mode'");
        int32_t modes[2 + 5 * kGenMaxBlocks];
        memcpy(modes, mode.data, mode.nbytes);
        if (gen_hybrid_layout(G, a.data(), modes, (int)(mode.nbytes / 4), &H) != 0)
            return r.fail(MWW_EMODEL, "model container: 'hy/mode' does not match the architecture (one entry per first conv, MixConv group, 1x1 conv, head; 0..2)");
        if ((size_t)H.sm_elems * 4 > 200 * 1024)
            return r.fail(MWW_EUNSUPPORTED, "model container: rings and quantisation buffers of one stream exceed 200 KB of shared memory");
        if (H.mode0) {
            if ((rc = r.get("hy/first_conv/w", kI8, k0f, &H.w0))) return rc;
            if ((rc = r.get("hy/first_conv/scale", kF32, G.c0, &H.s0))) return rc;
        }
        for (int i = 0; i < G.n_blocks; ++i) {
            if (H.any_dw[i]) {
                snprintf(name, sizeof name, "hy/b%d/dw/w", i); if ((rc = r.get(name, kI8, (size_t)G.kmax[i] * G.cin[i], &H.dw_w[i]))) return rc;
                snprintf(name, sizeof name, "hy/b%d/dw/scale", i); if ((rc = r.get(name, kF32, G.cin[i], &H.dw_s[i]))) return rc;
            }
            if (H.mode_pw[i]) {
                snprintf(name, sizeof name, "hy/b%d/pw/w", i); if ((rc = r.get(name, kI8, (size_t)G.cin[i] * G.cout[i], &H.pw_w[i]))) return rc;
                snprintf(name, sizeof name, "hy/b%d/pw/scale", i); if ((rc = r.get(name, kF32, G.cout[i], &H.pw_s[i]))) return rc;
            }
        }
        if (H.mode_head) {
            if ((rc = r.get("hy/head/w", kI8, (size_t)G.head_rows * G.c_last, &H.head_w))) return rc;
            if ((rc = r.get("hy/head/scale", kF32, 1, &H.head_s))) return rc;
        }
        return MWW_OK;
    }
    GenWeightsI8 &Q = m.GQ;
    if ((rc = r.get("q/first_conv/w", kI8, k0f, &Q.w0))) return rc;
    if ((rc = r.get("q/first_conv/bias", kI32, G.c0, &Q.b0))) return rc;
    if ((rc = r.get("q/first_conv/mult", kI32, G.c0, &Q.m0))) return rc;
    if ((rc = r.get("q/first_conv/shift", kI32, G.c0, &Q.s0))) return rc;
    for (int i = 0; i < G.n_blocks; ++i) {
        snprintf(name, sizeof name, "q/b%d/dw/w", i); if ((rc = r.get(name, kI8, (size_t)G.kmax[i] * G.cin[i], &Q.dw_w[i]))) return rc;
        snprintf(name, sizeof name, "q/b%d/dw/bias", i); if ((rc = r.get(name, kI32, G.cin[i], &Q.dw_b[i]))) return rc;
        snprintf(name, sizeof name, "q/b%d/dw/mult", i); if ((rc = r.get(name, kI32, G.cin[i], &Q.dw_m[i]))) return rc;
        snprintf(name, sizeof name, "q/b%d/dw/shift", i); if ((rc = r.get(name, kI32, G.cin[i], &Q.dw_s[i]))) return rc;
        snprintf(name, sizeof name, "q/b%d/pw/w", i); if ((rc = r.get(name, kI8, (size_t)G.cin[i] * G.cout[i], &Q.pw_w[i]))) return rc;
        snprintf(name, sizeof name, "q/b%d/pw/bias", i); if ((rc = r.get(name, kI32, G.cout[i], &Q.pw_b[i]))) return rc;
        snprintf(name, sizeof name, "q/b%d/pw/mult", i); if ((rc = r.get(name, kI32, G.cout[i], &Q.pw_m[i]))) return rc;
        snprintf(name, sizeof name, "q/b%d/pw/shift", i); if ((rc = r.get(name, kI32, G.cout[i], &Q.pw_s[i]))) return rc;
    }
    if ((rc = r.get("q/head/w", kI8, (size_t)G.head_rows * G.c_last, &Q.head_w))) return rc;
    if ((rc = r.get("q/logistic_lut", kI8, 256, &Q.lut))) return rc;
    if ((rc = r.scalar("q/head/bias", &Q.head_bias)) || (rc = r.scalar("q/head/mult", &Q.head_mult)) || (rc = r.scalar("q/head/shift", &Q.head_shift))) return rc;
    const size_t n_q = 4 + 2 * (size_t)G.n_blocks;       // in, first conv, (depthwise, pointwise) per block, logit, prob
    Tensor sc, zp;
    if (!find_tensor(blob, n, "q/scales", &sc) || sc.nbytes != n_q * 4 || !find_tensor(blob, n, "q/zps", &zp) || zp.nbytes != n_q * 4)
        return r.fail(MWW_EMODEL, std::string("model container: q/scales / q/zps must hold ") + (compiled ? "12" : "4 + 2 * n_blocks") + " entries");
    std::vector<float> scales(n_q);
    memcpy(scales.data(), sc.data, n_q * 4);
    memcpy(Q.zp, zp.data, n_q * 4);
    Q.in_scale = scales[0];
    m.in_scale = scales[0]; m.in_zp = Q.zp[0];
    m.out_scale = scales[n_q - 1]; m.out_zp = 0;      // uint8 output tensor: zero point -128 + 128 (utils.py:338)
    if (!compiled) return MWW_OK;
    // tensor-core operands: K-contiguous weight rows and zero-point-folded biases (mww_nn_i8_prep.h)
    const int8_t *pw_w[4];
    const int32_t *pw_b[4];
    for (int i = 0; i < 4; ++i) { pw_w[i] = r.host(Q.pw_w[i]); pw_b[i] = r.host(Q.pw_b[i]); }
    I8MmaOperands ops;
    build_i8_mma_operands(r.host(Q.w0), r.host(Q.b0), pw_w, pw_b, Q.zp, &ops);
    NnWeightsI8 &Wq = m.Wq;
    r.put(ops.w0t.data(), ops.w0t.size(), &Wq.w0t);
    r.put(ops.b0f.data(), ops.b0f.size() * 4, &Wq.b0f);
    for (int i = 0; i < 4; ++i) {
        r.put(ops.pwt[i].data(), ops.pwt[i].size(), &Wq.pwt[i]);
        r.put(ops.pw_bf[i].data(), ops.pw_bf[i].size() * 4, &Wq.pw_bf[i]);
    }
    if (getenv("MWW_NO_QLUT") == nullptr) {
        build_feature_qlut(Q.in_scale, Q.zp[0], &ops.qlut);
        r.put(ops.qlut.data(), ops.qlut.size(), &Wq.qlut);
    }
    return MWW_OK;
}

}  // namespace mww
