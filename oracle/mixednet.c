/*
 * oracle/mixednet.c -- CPU ORACLE (test infrastructure, NOT product code).
 *
 * Plain-C restatement of one streaming MixedNet invoke (what tf.lite.Interpreter.invoke()
 * executes at microwakeword/inference.py:113-119), fp32 and int8, batch 1, one stream per
 * object.  Topology: microwakeword/mixednet.py:307-386; ring semantics:
 * microwakeword/layers/stream.py:581-595 (concat(state, input) -> keep last N rows -> cell);
 * MixConv channel groups / StridedKeep: mixednet.py:132-136,197-231, strided_drop.py:80-84;
 * int8 contract: microwakeword/utils.py:289-348 executed with TFLite reference_integer_ops
 * semantics (SURVEY.md Appendix C).  Mirrors oracle/mixednet_ref.py (NumPy) so the two can
 * be cross-checked; this one is fast enough to be the timed CPU baseline.
 *
 *      *** PARITY UNPINNED *** (no TFLite / Keras / golden vectors exist here; SURVEY.md 8c)
 *
 * Weights come from the MWW container produced by tests/golden/make_golden.py
 * (layout documented in microwakeword_b200/model_file.py).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "mixednet.h"

#define NF 40
#define MAX_BLOCKS 8
#define MAX_CHANNELS 512                          /* per layer; the per-step buffers below hold this many */
#define MAX_KERNEL 64                             /* taps of the first conv (and so its largest stride), of a MixConv group, rows of the head */

struct tensor { const void *data; uint32_t dtype, ndim, shape[4]; uint64_t nbytes; };

struct dir_entry { char name[48]; uint32_t dtype, ndim, shape[4]; uint64_t offset, nbytes; };

static int find_tensor(const uint8_t *blob, size_t n, const char *name, struct tensor *out) {
    if (n < 24 || memcmp(blob, "MWWB200", 8) != 0) return 0;
    uint32_t hdr[4];
    memcpy(hdr, blob + 8, 16);
    const uint32_t count = hdr[1], dir_off = hdr[2];
    for (uint32_t i = 0; i < count; ++i) {
        struct dir_entry e;
        if ((size_t)dir_off + (i + 1) * sizeof e > n) return 0;
        memcpy(&e, blob + dir_off + i * sizeof e, sizeof e);
        if (strncmp(e.name, name, 48) == 0) {
            if (e.offset + e.nbytes > n) return 0;
            out->data = blob + e.offset; out->dtype = e.dtype; out->ndim = e.ndim;
            memcpy(out->shape, e.shape, sizeof e.shape); out->nbytes = e.nbytes;
            return 1;
        }
    }
    return 0;
}

struct block {
    int cin, cout, kmax;
    const float *dw_w, *dw_b, *pw_w, *pw_b;
    float *ring;                                   /* [kmax-1][cin] oldest first */
    /* int8 */
    const int8_t *qdw_w, *qpw_w;
    const int32_t *qdw_bias, *qdw_mult, *qdw_shift, *qpw_bias, *qpw_mult, *qpw_shift;
    int8_t *qring;
};

struct mwwo_mixednet {
    uint8_t *blob; size_t blob_n;
    int quantized;
    int c0, k0, stride, n_blocks, head_rows, ring0;
    const float *w0, *head_w, *head_b;
    float *ring_first;                             /* [ring0][40] */
    float *ring_head;                              /* [head_rows-1][c_last] */
    struct block blk[MAX_BLOCKS];
    /* int8 */
    const int8_t *qw0, *qhead_w, *qlut;
    const int32_t *qb0, *qm0, *qs0, *qhead_bias, *qhead_mult, *qhead_shift;
    const float *qscales; const int32_t *qzps;
    int8_t *qring_first, *qring_head;
};

static const void *need(struct mwwo_mixednet *m, const char *name, int *ok) {
    struct tensor t;
    if (!find_tensor(m->blob, m->blob_n, name, &t)) { *ok = 0; return NULL; }
    return t.data;
}

mwwo_mixednet *mwwo_mixednet_create(const void *blob, size_t n) {
    mwwo_mixednet *m = (mwwo_mixednet *)calloc(1, sizeof *m);
    if (!m) return NULL;
    m->blob = (uint8_t *)malloc(n);
    if (!m->blob) { free(m); return NULL; }
    memcpy(m->blob, blob, n);
    m->blob_n = n;
    struct tensor arch;
    if (!find_tensor(m->blob, n, "arch", &arch)) { mwwo_mixednet_free(m); return NULL; }
    const int32_t *a = (const int32_t *)arch.data;
    const size_t n_arch = arch.nbytes / 4;
    /* a model outside what the fixed-size step buffers hold is refused, never run */
    if (n_arch < 6) { mwwo_mixednet_free(m); return NULL; }
    m->c0 = a[0]; m->k0 = a[1]; m->stride = a[2]; m->n_blocks = a[4]; m->head_rows = a[5];
    if (a[3] != NF || m->n_blocks < 1 || m->n_blocks > MAX_BLOCKS || n_arch < 6 + 6 * (size_t)m->n_blocks ||
        m->c0 < 1 || m->c0 > MAX_CHANNELS || m->k0 < 1 || m->k0 > MAX_KERNEL || m->stride < 1 || m->stride > m->k0 ||
        m->head_rows < 1 || m->head_rows > MAX_KERNEL) { mwwo_mixednet_free(m); return NULL; }
    for (int i = 0; i < m->n_blocks; ++i) {
        const int32_t *e = a + 6 + 6 * i;
        if (e[0] < 1 || e[0] > MAX_CHANNELS || e[1] < 1 || e[1] > 4) { mwwo_mixednet_free(m); return NULL; }
        for (int j = 0; j < e[1]; ++j)
            if (e[2 + j] < 1 || e[2 + j] > MAX_KERNEL) { mwwo_mixednet_free(m); return NULL; }
    }
    m->ring0 = m->k0 - 1 - (m->stride - 1);
    struct tensor probe;
    m->quantized = find_tensor(m->blob, n, "q/scales", &probe);
    int ok = 1;
    char name[64];
    int cin = m->c0;
    for (int i = 0; i < m->n_blocks; ++i) {
        struct block *b = &m->blk[i];
        const int32_t *e = a + 6 + 6 * i;
        b->cin = cin; b->cout = e[0]; b->kmax = 0;
        for (int j = 0; j < e[1]; ++j) if (e[2 + j] > b->kmax) b->kmax = e[2 + j];
        if (m->quantized) {
            snprintf(name, sizeof name, "q/b%d/dw/w", i); b->qdw_w = (const int8_t *)need(m, name, &ok);
            snprintf(name, sizeof name, "q/b%d/dw/bias", i); b->qdw_bias = (const int32_t *)need(m, name, &ok);
            snprintf(name, sizeof name, "q/b%d/dw/mult", i); b->qdw_mult = (const int32_t *)need(m, name, &ok);
            snprintf(name, sizeof name, "q/b%d/dw/shift", i); b->qdw_shift = (const int32_t *)need(m, name, &ok);
            snprintf(name, sizeof name, "q/b%d/pw/w", i); b->qpw_w = (const int8_t *)need(m, name, &ok);
            snprintf(name, sizeof name, "q/b%d/pw/bias", i); b->qpw_bias = (const int32_t *)need(m, name, &ok);
            snprintf(name, sizeof name, "q/b%d/pw/mult", i); b->qpw_mult = (const int32_t *)need(m, name, &ok);
            snprintf(name, sizeof name, "q/b%d/pw/shift", i); b->qpw_shift = (const int32_t *)need(m, name, &ok);
            b->qring = (int8_t *)calloc((size_t)(b->kmax - 1) * cin + 1, 1);
        } else {
            snprintf(name, sizeof name, "b%d/dw/w", i); b->dw_w = (const float *)need(m, name, &ok);
            snprintf(name, sizeof name, "b%d/dw/b", i); b->dw_b = (const float *)need(m, name, &ok);
            snprintf(name, sizeof name, "b%d/pw/w", i); b->pw_w = (const float *)need(m, name, &ok);
            snprintf(name, sizeof name, "b%d/pw/b", i); b->pw_b = (const float *)need(m, name, &ok);
            b->ring = (float *)calloc((size_t)(b->kmax - 1) * cin + 1, sizeof(float));
        }
        cin = b->cout;
    }
    if (m->quantized) {
        m->qw0 = (const int8_t *)need(m, "q/first_conv/w", &ok);
        m->qb0 = (const int32_t *)need(m, "q/first_conv/bias", &ok);
        m->qm0 = (const int32_t *)need(m, "q/first_conv/mult", &ok);
        m->qs0 = (const int32_t *)need(m, "q/first_conv/shift", &ok);
        m->qhead_w = (const int8_t *)need(m, "q/head/w", &ok);
        m->qhead_bias = (const int32_t *)need(m, "q/head/bias", &ok);
        m->qhead_mult = (const int32_t *)need(m, "q/head/mult", &ok);
        m->qhead_shift = (const int32_t *)need(m, "q/head/shift", &ok);
        m->qlut = (const int8_t *)need(m, "q/logistic_lut", &ok);
        m->qscales = (const float *)need(m, "q/scales", &ok);
        m->qzps = (const int32_t *)need(m, "q/zps", &ok);
        m->qring_first = (int8_t *)calloc((size_t)m->ring0 * NF + 1, 1);
        m->qring_head = (int8_t *)calloc((size_t)(m->head_rows - 1) * cin + 1, 1);
    } else {
        m->w0 = (const float *)need(m, "first_conv/w", &ok);
        m->head_w = (const float *)need(m, "head/w", &ok);
        m->head_b = (const float *)need(m, "head/b", &ok);
        m->ring_first = (float *)calloc((size_t)m->ring0 * NF + 1, sizeof(float));
        m->ring_head = (float *)calloc((size_t)(m->head_rows - 1) * cin + 1, sizeof(float));
    }
    if (!ok) { mwwo_mixednet_free(m); return NULL; }
    mwwo_mixednet_reset(m);
    return m;
}

void mwwo_mixednet_free(mwwo_mixednet *m) {
    if (!m) return;
    for (int i = 0; i < MAX_BLOCKS; ++i) { free(m->blk[i].ring); free(m->blk[i].qring); }
    free(m->ring_first); free(m->ring_head); free(m->qring_first); free(m->qring_head);
    free(m->blob); free(m);
}

int mwwo_mixednet_is_quantized(const mwwo_mixednet *m) { return m->quantized; }
int mwwo_mixednet_stride(const mwwo_mixednet *m) { return m->stride; }
float mwwo_mixednet_input_scale(const mwwo_mixednet *m) { return m->quantized ? m->qscales[0] : 0.f; }
int mwwo_mixednet_input_zero_point(const mwwo_mixednet *m) { return m->quantized ? m->qzps[0] : 0; }

void mwwo_mixednet_reset(mwwo_mixednet *m) {
    const int c_last = m->blk[m->n_blocks - 1].cout;
    if (m->quantized) {
        /* quantised state variables hold the zero POINT (real 0) of the tensor they buffer */
        memset(m->qring_first, (int8_t)m->qzps[0], (size_t)m->ring0 * NF);
        for (int i = 0; i < m->n_blocks; ++i)
            memset(m->blk[i].qring, (int8_t)m->qzps[1 + 2 * i], (size_t)(m->blk[i].kmax - 1) * m->blk[i].cin);
        memset(m->qring_head, (int8_t)m->qzps[1 + 2 * m->n_blocks], (size_t)(m->head_rows - 1) * c_last);
    } else {
        memset(m->ring_first, 0, sizeof(float) * m->ring0 * NF);
        for (int i = 0; i < m->n_blocks; ++i)
            memset(m->blk[i].ring, 0, sizeof(float) * (m->blk[i].kmax - 1) * m->blk[i].cin);
        memset(m->ring_head, 0, sizeof(float) * (m->head_rows - 1) * c_last);
    }
}

/* ------------------------------------------------------------------------- */
/* fp32 invoke                                                               */

float mwwo_mixednet_step_f32(mwwo_mixednet *m, const float *x /* [stride][40] */, float *logit_out) {
    float mem[MAX_KERNEL * NF];         /* concat(state, input) of the first conv: k0 rows */
    float a[MAX_CHANNELS], d[MAX_CHANNELS], nxt[MAX_CHANNELS];
    const int k0 = m->k0, c0 = m->c0;
    memcpy(mem, m->ring_first, sizeof(float) * m->ring0 * NF);
    memcpy(mem + m->ring0 * NF, x, sizeof(float) * m->stride * NF);
    if (m->ring0) memcpy(m->ring_first, mem + (k0 - m->ring0) * NF, sizeof(float) * m->ring0 * NF);
    for (int o = 0; o < c0; ++o) {
        float acc = 0.f;
        for (int k = 0; k < k0; ++k)
            for (int f = 0; f < NF; ++f) acc += mem[k * NF + f] * m->w0[(k * NF + f) * c0 + o];
        a[o] = acc > 0.f ? acc : 0.f;
    }
    for (int i = 0; i < m->n_blocks; ++i) {
        struct block *b = &m->blk[i];
        const int rows = b->kmax - 1, cin = b->cin, cout = b->cout;
        /* depthwise over concat(ring, new row); weights are zero padded for the shorter kernels */
        for (int c = 0; c < cin; ++c) {
            float acc = 0.f;
            for (int k = 0; k < rows; ++k) acc += b->ring[k * cin + c] * b->dw_w[k * cin + c];
            acc += a[c] * b->dw_w[rows * cin + c];
            d[c] = acc + b->dw_b[c];
        }
        /* ring <- last (kmax-1) rows of the concat */
        if (rows > 0) {                            /* a 1-tap kernel keeps no history */
            memmove(b->ring, b->ring + cin, sizeof(float) * (rows - 1) * cin);
            memcpy(b->ring + (rows - 1) * cin, a, sizeof(float) * cin);
        }
        for (int o = 0; o < cout; ++o) {
            float acc = 0.f;
            for (int c = 0; c < cin; ++c) acc += d[c] * b->pw_w[c * cout + o];
            acc += b->pw_b[o];
            nxt[o] = acc > 0.f ? acc : 0.f;
        }
        memcpy(a, nxt, sizeof(float) * cout);
    }
    const int c_last = m->blk[m->n_blocks - 1].cout, hr = m->head_rows - 1;
    float acc = 0.f;
    for (int k = 0; k < hr; ++k)
        for (int c = 0; c < c_last; ++c) acc += m->ring_head[k * c_last + c] * m->head_w[k * c_last + c];
    for (int c = 0; c < c_last; ++c) acc += a[c] * m->head_w[hr * c_last + c];
    if (hr > 0) {
        memmove(m->ring_head, m->ring_head + c_last, sizeof(float) * (hr - 1) * c_last);
        memcpy(m->ring_head + (hr - 1) * c_last, a, sizeof(float) * c_last);
    }
    const float logit = acc + m->head_b[0];
    if (logit_out) *logit_out = logit;
    return 1.0f / (1.0f + expf(-logit));
}

/* ------------------------------------------------------------------------- */
/* int8 invoke (TFLite reference integer kernels)                            */

static int32_t srdhm(int32_t a, int32_t b) {
    if (a == INT32_MIN && b == INT32_MIN) return INT32_MAX;
    const int64_t ab = (int64_t)a * (int64_t)b;
    const int32_t nudge = ab >= 0 ? (1 << 30) : (1 - (1 << 30));
    return (int32_t)((ab + nudge) / (1ll << 31));       /* C division: truncation toward zero */
}
static int32_t rdbp(int32_t x, int exponent) {
    const int32_t mask = (int32_t)((1ll << exponent) - 1);
    const int32_t rem = x & mask;
    const int32_t thr = (mask >> 1) + (x < 0 ? 1 : 0);
    return (x >> exponent) + (rem > thr ? 1 : 0);
}
static int32_t mbqm(int32_t x, int32_t mult, int shift) {
    const int left = shift > 0 ? shift : 0, right = shift > 0 ? 0 : -shift;
    return rdbp(srdhm(x * (1 << left), mult), right);
}
static int8_t requant(int32_t acc, int32_t mult, int shift, int zp_out, int relu) {
    int32_t y = mbqm(acc, mult, shift) + zp_out;
    const int lo = relu ? zp_out : -128;
    if (y < lo) y = lo;
    if (y > 127) y = 127;
    return (int8_t)y;
}

int mwwo_mixednet_step_int8(mwwo_mixednet *m, const int8_t *x /* [stride][40] */, int *logit_out) {
    int8_t mem[MAX_KERNEL * NF], a[MAX_CHANNELS], d[MAX_CHANNELS], nxt[MAX_CHANNELS];
    const int k0 = m->k0, c0 = m->c0;
    const int32_t *zp = m->qzps;
    memcpy(mem, m->qring_first, (size_t)m->ring0 * NF);
    memcpy(mem + m->ring0 * NF, x, (size_t)m->stride * NF);
    if (m->ring0) memcpy(m->qring_first, mem + (k0 - m->ring0) * NF, (size_t)m->ring0 * NF);
    for (int o = 0; o < c0; ++o) {
        int32_t acc = 0;
        for (int k = 0; k < k0; ++k)
            for (int f = 0; f < NF; ++f) acc += ((int32_t)mem[k * NF + f] - zp[0]) * m->qw0[(k * NF + f) * c0 + o];
        acc += m->qb0[o];
        a[o] = requant(acc, m->qm0[o], m->qs0[o], zp[1], 1);
    }
    for (int i = 0; i < m->n_blocks; ++i) {
        struct block *b = &m->blk[i];
        const int rows = b->kmax - 1, cin = b->cin, cout = b->cout;
        const int zp_in = zp[1 + 2 * i], zp_d = zp[2 + 2 * i], zp_p = zp[3 + 2 * i];
        for (int c = 0; c < cin; ++c) {
            int32_t acc = 0;
            for (int k = 0; k < rows; ++k) acc += ((int32_t)b->qring[k * cin + c] - zp_in) * b->qdw_w[k * cin + c];
            acc += ((int32_t)a[c] - zp_in) * b->qdw_w[rows * cin + c];
            acc += b->qdw_bias[c];
            d[c] = requant(acc, b->qdw_mult[c], b->qdw_shift[c], zp_d, 0);
        }
        if (rows > 0) {
            memmove(b->qring, b->qring + cin, (size_t)(rows - 1) * cin);
            memcpy(b->qring + (rows - 1) * cin, a, (size_t)cin);
        }
        for (int o = 0; o < cout; ++o) {
            int32_t acc = 0;
            for (int c = 0; c < cin; ++c) acc += ((int32_t)d[c] - zp_d) * b->qpw_w[c * cout + o];
            acc += b->qpw_bias[o];
            nxt[o] = requant(acc, b->qpw_mult[o], b->qpw_shift[o], zp_p, 1);
        }
        memcpy(a, nxt, (size_t)cout);
    }
    const int c_last = m->blk[m->n_blocks - 1].cout, hr = m->head_rows - 1;
    const int zp_in = zp[1 + 2 * m->n_blocks], zp_fc = zp[2 + 2 * m->n_blocks];
    int32_t acc = 0;
    for (int k = 0; k < hr; ++k)
        for (int c = 0; c < c_last; ++c) acc += ((int32_t)m->qring_head[k * c_last + c] - zp_in) * m->qhead_w[k * c_last + c];
    for (int c = 0; c < c_last; ++c) acc += ((int32_t)a[c] - zp_in) * m->qhead_w[hr * c_last + c];
    if (hr > 0) {
        memmove(m->qring_head, m->qring_head + c_last, (size_t)(hr - 1) * c_last);
        memcpy(m->qring_head + (hr - 1) * c_last, a, (size_t)c_last);
    }
    acc += m->qhead_bias[0];
    const int8_t logit = requant(acc, m->qhead_mult[0], m->qhead_shift[0], zp_fc, 0);
    if (logit_out) *logit_out = logit;
    return (int)m->qlut[(uint8_t)logit] + 128;       /* LOGISTIC LUT, then QUANTIZE int8 -> uint8 */
}

/* ------------------------------------------------------------------------- */
/* predict_spectrogram loop (inference.py:98-123) over uint16 features        */

size_t mwwo_mixednet_predict_u16(mwwo_mixednet *m, const uint16_t *feat, size_t rows, float *probs, size_t max_probs) {
    const int s = m->stride;
    size_t n = 0;
    float xf[MAX_KERNEL * NF];                     /* one step's rows: stride <= k0 <= MAX_KERNEL */
    int8_t xq[MAX_KERNEL * NF];
    for (size_t last = (size_t)s; last <= rows; last += (size_t)s) {
        const uint16_t *chunk = feat + (last - s) * NF;
        for (int i = 0; i < s * NF; ++i) xf[i] = (float)chunk[i] * 0.0390625f;      /* inference.py:94 */
        float p;
        if (m->quantized) {
            const float scale = m->qscales[0];
            const float zp = (float)m->qzps[0];
            for (int i = 0; i < s * NF; ++i) xq[i] = (int8_t)(int32_t)(xf[i] / scale + zp);   /* inference.py:146-147 */
            p = (1.0f / 255.0f) * (float)mwwo_mixednet_step_int8(m, xq, NULL);        /* inference.py:162-170 */
        } else {
            p = mwwo_mixednet_step_f32(m, xf, NULL);
        }
        if (n < max_probs) probs[n] = p;
        ++n;
    }
    return n;
}
