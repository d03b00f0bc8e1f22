/*
 * tests/hybrid_ref/hybrid_ref.c -- CPU ORACLE for hybrid models (test infrastructure, NOT product code).
 *
 * The float streaming .tflite the reference writes with quantize=False (utils.py:289-348: Optimize.DEFAULT without a
 * representative dataset = dynamic-range quantisation) stores the weights of large CONV_2D / DEPTHWISE_CONV_2D /
 * FULLY_CONNECTED ops as symmetric per-channel int8, and tf.lite.Interpreter runs those ops with its HYBRID kernels.  This
 * file restates one streaming invoke of such a model (batch 1, one stream per object) over an MWW container with hy/
 * tensors (layout: microwakeword_b200/model_file.py).  Topology and ring semantics are those of oracle/mixednet.c; a
 * container without hy/mode is refused (plain fp32 models belong to oracle/mixednet.c).
 *
 * [UPSTREAM-RECALL]  TFLite's hybrid kernels, restated from knowledge of the public sources (not vendored, not pinned):
 * tensorflow/lite/kernels/internal/portable_tensor_utils.cc AsymmetricQuantizeFloats / SymmetricQuantizeFloats,
 * conv.cc EvalHybridPerChannel, depthwise_conv.cc EvalHybridPerChannel, fully_connected.cc EvalHybrid.  On every invoke
 * each hybrid op quantises its whole float input tensor to int8, accumulates int8 x int8 in int32 and rescales to float.
 * The float operation order of the rescale is not pinned by TFLite (kernel variant, delegates); this file fixes one order
 * per op and the GPU kernel (microwakeword_b200/csrc/mww_nn_generic.cuh, gen_hy_*) reproduces it operation for operation.
 * Float layers of a hybrid model use fmaf in the loop order of the generic fp32 phases.  DESIGN.md section 0 lists the
 * choices.  Built with -ffp-contract=off: every float operation below rounds once, where it is written.
 */
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#define NF 40
#define MAX_BLOCKS 8
#define MAX_CHANNELS 512                           /* per layer; the per-step buffers of hyref_step hold this many */
#define MAX_KERNEL 64                              /* taps of the first conv (and so its largest stride), of a MixConv group, head rows */

struct tensor { const void *data; uint32_t dtype, nbytes; };
struct dir_entry { char name[48]; uint32_t dtype, ndim, shape[4]; uint64_t offset, nbytes; };

static int find_tensor(const uint8_t *blob, size_t n, const char *name, struct tensor *out) {
    if (n < 24 || memcmp(blob, "MWWB200", 8) != 0) return 0;
    uint32_t hdr[4];
    memcpy(hdr, blob + 8, 16);
    for (uint32_t i = 0; i < hdr[1]; ++i) {
        struct dir_entry e;
        if ((size_t)hdr[2] + (i + 1) * sizeof e > n) return 0;
        memcpy(&e, blob + hdr[2] + i * sizeof e, sizeof e);
        if (strncmp(e.name, name, 48) == 0) {
            if (e.offset + e.nbytes > n) return 0;
            out->data = blob + e.offset; out->dtype = e.dtype; out->nbytes = (uint32_t)e.nbytes;
            return 1;
        }
    }
    return 0;
}

struct block {
    int cin, cout, kmax;
    const float *dw_w, *dw_b, *pw_w, *pw_b;
    float *ring;                                   /* [kmax-1][cin] oldest first */
    int n_groups, gk[4], gc0[4], gn[4], gmode[4], pw_mode;
    const int8_t *hdw_w, *hpw_w;
    const float *hdw_s, *hpw_s;
};

typedef struct hyref {
    uint8_t *blob; size_t blob_n;
    int c0, k0, stride, n_blocks, head_rows, ring0;
    const float *w0, *head_w, *head_b;
    float *ring_first, *ring_head;
    struct block blk[MAX_BLOCKS];
    int mode0, head_mode;
    const int8_t *hw0, *hhead_w;
    const float *hs0, *hhead_s;
    float *hx;                                     /* one op's float input tensor, gathered */
    int8_t *hq;                                    /* ... and its int8 codes */
} hyref;

static const void *need(hyref *m, const char *name, int *ok) {
    struct tensor t;
    if (!find_tensor(m->blob, m->blob_n, name, &t)) { *ok = 0; return NULL; }
    return t.data;
}

void hyref_free(hyref *m) {
    if (!m) return;
    for (int i = 0; i < MAX_BLOCKS; ++i) free(m->blk[i].ring);
    free(m->ring_first); free(m->ring_head); free(m->hx); free(m->hq); free(m->blob); free(m);
}

void hyref_reset(hyref *m) {
    memset(m->ring_first, 0, sizeof(float) * m->ring0 * NF);
    for (int i = 0; i < m->n_blocks; ++i) memset(m->blk[i].ring, 0, sizeof(float) * (m->blk[i].kmax - 1) * m->blk[i].cin);
    memset(m->ring_head, 0, sizeof(float) * (m->head_rows - 1) * m->blk[m->n_blocks - 1].cout);
}

/* hy/mode: one entry per op -- first conv, per block its MixConv groups then its 1x1 conv, head -- 0 float, 1 hybrid with
 * asymmetric input quantisation, 2 hybrid with symmetric.  NULL on a malformed container or one without hy/mode. */
hyref *hyref_create(const void *blob, size_t n) {
    hyref *m = (hyref *)calloc(1, sizeof *m);
    if (!m) return NULL;
    m->blob = (uint8_t *)malloc(n);
    if (!m->blob) { free(m); return NULL; }
    memcpy(m->blob, blob, n);
    m->blob_n = n;
    struct tensor arch, mt;
    if (!find_tensor(m->blob, n, "arch", &arch) || !find_tensor(m->blob, n, "hy/mode", &mt)) { hyref_free(m); return NULL; }
    const int32_t *a = (const int32_t *)arch.data;
    const int n_arch = (int)(arch.nbytes / 4);
    m->c0 = a[0]; m->k0 = a[1]; m->stride = a[2]; m->n_blocks = a[4]; m->head_rows = a[5];
    if (a[3] != NF || m->n_blocks < 1 || m->n_blocks > MAX_BLOCKS || n_arch < 6 + 6 * m->n_blocks) { hyref_free(m); return NULL; }
    /* a model outside what the fixed-size step buffers hold is refused, never run */
    if (m->c0 < 1 || m->c0 > MAX_CHANNELS || m->k0 < 1 || m->k0 > MAX_KERNEL || m->stride < 1 || m->stride > m->k0 ||
        m->head_rows < 1 || m->head_rows > MAX_KERNEL) { hyref_free(m); return NULL; }
    for (int i = 0; i < m->n_blocks; ++i) {
        const int32_t *e = a + 6 + 6 * i;
        if (e[0] < 1 || e[0] > MAX_CHANNELS || e[1] < 1 || e[1] > 4) { hyref_free(m); return NULL; }
        for (int j = 0; j < e[1]; ++j)
            if (e[2 + j] < 1 || e[2 + j] > MAX_KERNEL) { hyref_free(m); return NULL; }
    }
    m->ring0 = m->k0 - m->stride;
    int n_slots = 2;
    for (int i = 0; i < m->n_blocks; ++i) n_slots += a[6 + 6 * i + 1] + 1;
    int32_t mode[2 + MAX_BLOCKS * 5];
    if (mt.dtype != 2 || mt.nbytes != (uint32_t)n_slots * 4 || n_slots > 2 + MAX_BLOCKS * 5) { hyref_free(m); return NULL; }
    memcpy(mode, mt.data, mt.nbytes);
    for (int i = 0; i < n_slots; ++i) if (mode[i] < 0 || mode[i] > 2) { hyref_free(m); return NULL; }
    int ok = 1, s = 0;
    char name[64];
    size_t max_in = (size_t)m->k0 * NF;
    m->w0 = (const float *)need(m, "first_conv/w", &ok);
    m->mode0 = mode[s++];
    if (m->mode0) { m->hw0 = (const int8_t *)need(m, "hy/first_conv/w", &ok); m->hs0 = (const float *)need(m, "hy/first_conv/scale", &ok); }
    int cin = m->c0;
    for (int i = 0; i < m->n_blocks; ++i) {
        struct block *b = &m->blk[i];
        const int32_t *e = a + 6 + 6 * i;
        b->cin = cin; b->cout = e[0]; b->kmax = 0;
        b->n_groups = e[1];
        int c = 0, any = 0;
        for (int j = 0; j < b->n_groups; ++j) {
            b->gk[j] = e[2 + j];
            if (b->gk[j] > b->kmax) b->kmax = b->gk[j];
            b->gn[j] = cin / b->n_groups + (j == 0 ? cin % b->n_groups : 0);        /* mixednet.py:132-136 */
            b->gc0[j] = c; c += b->gn[j];
            b->gmode[j] = mode[s++];
            any |= b->gmode[j];
            if ((size_t)b->gk[j] * b->gn[j] > max_in) max_in = (size_t)b->gk[j] * b->gn[j];
        }
        b->pw_mode = mode[s++];
        snprintf(name, sizeof name, "b%d/dw/w", i); b->dw_w = (const float *)need(m, name, &ok);
        snprintf(name, sizeof name, "b%d/dw/b", i); b->dw_b = (const float *)need(m, name, &ok);
        snprintf(name, sizeof name, "b%d/pw/w", i); b->pw_w = (const float *)need(m, name, &ok);
        snprintf(name, sizeof name, "b%d/pw/b", i); b->pw_b = (const float *)need(m, name, &ok);
        if (any) {
            snprintf(name, sizeof name, "hy/b%d/dw/w", i); b->hdw_w = (const int8_t *)need(m, name, &ok);
            snprintf(name, sizeof name, "hy/b%d/dw/scale", i); b->hdw_s = (const float *)need(m, name, &ok);
        }
        if (b->pw_mode) {
            snprintf(name, sizeof name, "hy/b%d/pw/w", i); b->hpw_w = (const int8_t *)need(m, name, &ok);
            snprintf(name, sizeof name, "hy/b%d/pw/scale", i); b->hpw_s = (const float *)need(m, name, &ok);
        }
        if ((size_t)cin > max_in) max_in = (size_t)cin;
        b->ring = (float *)calloc((size_t)(b->kmax - 1) * cin + 1, sizeof(float));
        if (!b->ring) ok = 0;
        cin = b->cout;
    }
    m->head_w = (const float *)need(m, "head/w", &ok);
    m->head_b = (const float *)need(m, "head/b", &ok);
    m->head_mode = mode[s++];
    if (m->head_mode) { m->hhead_w = (const int8_t *)need(m, "hy/head/w", &ok); m->hhead_s = (const float *)need(m, "hy/head/scale", &ok); }
    if ((size_t)m->head_rows * cin > max_in) max_in = (size_t)m->head_rows * cin;
    m->ring_first = (float *)calloc((size_t)m->ring0 * NF + 1, sizeof(float));
    m->ring_head = (float *)calloc((size_t)(m->head_rows - 1) * cin + 1, sizeof(float));
    m->hx = (float *)malloc(max_in * sizeof(float));
    m->hq = (int8_t *)malloc(max_in);
    if (!ok || !m->ring_first || !m->ring_head || !m->hx || !m->hq) { hyref_free(m); return NULL; }
    hyref_reset(m);
    return m;
}

int hyref_stride(const hyref *m) { return m->stride; }

size_t hyref_get_state(const hyref *m, float *out, size_t max_elems) {
    const int c_last = m->blk[m->n_blocks - 1].cout;
    size_t n = 0;
#define PUT(src, cnt) do { const size_t c_ = (size_t)(cnt); if (out && n + c_ <= max_elems) memcpy(out + n, (src), sizeof(float) * c_); n += c_; } while (0)
    PUT(m->ring_first, (size_t)m->ring0 * NF);
    for (int i = 0; i < m->n_blocks; ++i) PUT(m->blk[i].ring, (size_t)(m->blk[i].kmax - 1) * m->blk[i].cin);
    PUT(m->ring_head, (size_t)(m->head_rows - 1) * c_last);
#undef PUT
    return n;
}

/* ---- [UPSTREAM-RECALL] input quantisers ---- */
static void quantize_asym(const float *x, int n, int8_t *q, float *scale_out, int32_t *zp_out) {
    float mn = x[0], mx = x[0];
    for (int i = 1; i < n; ++i) { if (x[i] < mn) mn = x[i]; if (x[i] > mx) mx = x[i]; }
    const double rmin = fmin(0.0, (double)mn), rmax = fmax(0.0, (double)mx);
    if (rmin == rmax) { memset(q, 0, (size_t)n); *scale_out = 1.0f; *zp_out = 0; return; }
    const double qmin = -128.0, qmax = 127.0;
    const double scale = (rmax - rmin) / (qmax - qmin);
    const double zp_from_min = qmin - rmin / scale, zp_from_max = qmax - rmax / scale;
    const double err_min = fabs(qmin) + fabs(rmin / scale), err_max = fabs(qmax) + fabs(rmax / scale);
    const double zp_d = err_min < err_max ? zp_from_min : zp_from_max;
    int32_t zp;
    if (zp_d <= qmin) zp = -128;
    else if (zp_d >= qmax) zp = 127;
    else zp = (int32_t)round(zp_d);
    const float sf = (float)scale, inv = 1.0f / sf;
    for (int i = 0; i < n; ++i) {
        const int32_t v = (int32_t)roundf((float)zp + x[i] * inv);
        q[i] = (int8_t)(v < -128 ? -128 : (v > 127 ? 127 : v));
    }
    *scale_out = sf; *zp_out = zp;
}
static void quantize_sym(const float *x, int n, int8_t *q, float *scale_out) {
    float mn = x[0], mx = x[0];
    for (int i = 1; i < n; ++i) { if (x[i] < mn) mn = x[i]; if (x[i] > mx) mx = x[i]; }
    const float range = fmaxf(fabsf(mn), fabsf(mx));
    if (range == 0.0f) { memset(q, 0, (size_t)n); *scale_out = 1.0f; return; }
    const float inv = 127.0f / range;
    for (int i = 0; i < n; ++i) {
        const int32_t v = (int32_t)roundf(x[i] * inv);
        q[i] = (int8_t)(v < -127 ? -127 : (v > 127 ? 127 : v));
    }
    *scale_out = range / 127.0f;
}
/* mode 1 asymmetric, 2 symmetric (zero point 0) */
void hyref_quantize(int mode, const float *x, int n, int8_t *q, float *scale, int32_t *zp) {
    if (mode == 2) { quantize_sym(x, n, q, scale); *zp = 0; }
    else quantize_asym(x, n, q, scale, zp);
}

/* CONV_2D / DEPTHWISE_CONV_2D per-channel epilogue: (float)acc * w_scale[c] * input_scale + bias[c], left to right */
static float conv_out(int32_t acc, float w_scale, float in_scale, float bias) {
    float y = (float)acc * w_scale;
    y = y * in_scale;
    return y + bias;
}

float hyref_step(hyref *m, const float *x /* [stride][40] */, float *logit_out) {
    float mem[MAX_KERNEL * NF], a[MAX_CHANNELS], d[MAX_CHANNELS], nxt[MAX_CHANNELS];
    const int k0 = m->k0, c0 = m->c0;
    float *hx = m->hx;
    int8_t *hq = m->hq;
    float sc;
    int32_t zp;
    memcpy(mem, m->ring_first, sizeof(float) * m->ring0 * NF);
    memcpy(mem + m->ring0 * NF, x, sizeof(float) * m->stride * NF);
    if (m->ring0) memcpy(m->ring_first, mem + (k0 - m->ring0) * NF, sizeof(float) * m->ring0 * NF);
    /* first conv: input tensor = the [k0, 40] window */
    if (m->mode0) {
        hyref_quantize(m->mode0, mem, k0 * NF, hq, &sc, &zp);
        for (int o = 0; o < c0; ++o) {
            int32_t acc = 0;
            for (int k = 0; k < k0 * NF; ++k) acc += ((int32_t)hq[k] - zp) * m->hw0[k * c0 + o];
            const float y = conv_out(acc, m->hs0[o], sc, 0.0f);
            a[o] = y > 0.f ? y : 0.f;
        }
    } else {
        for (int o = 0; o < c0; ++o) {
            float acc = 0.f;
            for (int k = 0; k < k0 * NF; ++k) acc = fmaf(mem[k], m->w0[k * c0 + o], acc);
            a[o] = acc > 0.f ? acc : 0.f;
        }
    }
    for (int i = 0; i < m->n_blocks; ++i) {
        struct block *b = &m->blk[i];
        const int rows = b->kmax - 1, cin = b->cin, cout = b->cout, kmax = b->kmax;
        /* row r of the ring memory concat(ring, a): r < rows from the ring, r == rows the new row */
#define MEMV(r, c) ((r) < rows ? b->ring[(r) * cin + (c)] : a[c])
        for (int g = 0; g < b->n_groups; ++g) {
            const int k = b->gk[g], cs = b->gc0[g], cn = b->gn[g];
            if (b->gmode[g]) {
                /* input tensor of the group = the LAST k rows of the memory (StridedKeep), the group's channels */
                for (int r = 0; r < k; ++r)
                    for (int c = 0; c < cn; ++c) hx[r * cn + c] = MEMV(kmax - k + r, cs + c);
                hyref_quantize(b->gmode[g], hx, k * cn, hq, &sc, &zp);
                for (int c = 0; c < cn; ++c) {
                    int32_t acc = 0;
                    for (int r = 0; r < k; ++r) acc += ((int32_t)hq[r * cn + c] - zp) * b->hdw_w[(kmax - k + r) * cin + cs + c];
                    d[cs + c] = conv_out(acc, b->hdw_s[cs + c], sc, b->dw_b[cs + c]);
                }
            } else {
                for (int c = cs; c < cs + cn; ++c) {
                    float acc = 0.f;
                    for (int r = 0; r < kmax; ++r) acc = fmaf(MEMV(r, c), b->dw_w[r * cin + c], acc);
                    d[c] = acc + b->dw_b[c];
                }
            }
        }
#undef MEMV
        if (rows > 0) {
            memmove(b->ring, b->ring + cin, sizeof(float) * (rows - 1) * cin);
            memcpy(b->ring + (rows - 1) * cin, a, sizeof(float) * cin);
        }
        if (b->pw_mode) {
            hyref_quantize(b->pw_mode, d, cin, hq, &sc, &zp);
            for (int o = 0; o < cout; ++o) {
                int32_t acc = 0;
                for (int c = 0; c < cin; ++c) acc += ((int32_t)hq[c] - zp) * b->hpw_w[c * cout + o];
                const float y = conv_out(acc, b->hpw_s[o], sc, b->pw_b[o]);
                nxt[o] = y > 0.f ? y : 0.f;
            }
        } else {
            for (int o = 0; o < cout; ++o) {
                float acc = 0.f;
                for (int c = 0; c < cin; ++c) acc = fmaf(d[c], b->pw_w[c * cout + o], acc);
                acc += b->pw_b[o];
                nxt[o] = acc > 0.f ? acc : 0.f;
            }
        }
        memcpy(a, nxt, sizeof(float) * cout);
    }
    const int c_last = m->blk[m->n_blocks - 1].cout, hr = m->head_rows - 1;
    /* head input tensor = the flattened [head_rows, c_last] ring memory */
    memcpy(hx, m->ring_head, sizeof(float) * hr * c_last);
    memcpy(hx + hr * c_last, a, sizeof(float) * c_last);
    float logit;
    if (m->head_mode) {
        hyref_quantize(m->head_mode, hx, (hr + 1) * c_last, hq, &sc, &zp);
        int32_t acc = 0;
        for (int e = 0; e < (hr + 1) * c_last; ++e) acc += ((int32_t)hq[e] - zp) * m->hhead_w[e];
        /* FULLY_CONNECTED: output starts at the bias, += (float)acc * (input_scale * weight_scale) */
        const float s = sc * m->hhead_s[0];
        logit = m->head_b[0] + (float)acc * s;
    } else {
        float acc = 0.f;
        for (int c = 0; c < c_last; ++c) {
            float p = 0.f;
            for (int k = 0; k <= hr; ++k) p = fmaf(hx[k * c_last + c], m->head_w[k * c_last + c], p);
            acc += p;
        }
        logit = acc + m->head_b[0];
    }
    if (hr > 0) {
        memmove(m->ring_head, m->ring_head + c_last, sizeof(float) * (hr - 1) * c_last);
        memcpy(m->ring_head + (hr - 1) * c_last, a, sizeof(float) * c_last);
    }
    if (logit_out) *logit_out = logit;
    return 1.0f / (1.0f + expf(-logit));
}

/* Model.predict_spectrogram over uint16 features (stride == input_feature_slices, inference.py:98-123); returns #probs */
size_t hyref_predict_u16(hyref *m, const uint16_t *feat, size_t rows, float *probs, size_t max_probs) {
    const int s = m->stride;
    size_t n = 0;
    float xf[MAX_KERNEL * NF];
    for (size_t last = (size_t)s; last <= rows; last += (size_t)s) {
        const uint16_t *chunk = feat + (last - s) * NF;
        for (int i = 0; i < s * NF; ++i) xf[i] = (float)chunk[i] * 0.0390625f;      /* inference.py:94 */
        const float p = hyref_step(m, xf, NULL);
        if (n < max_probs) probs[n] = p;
        ++n;
    }
    return n;
}
