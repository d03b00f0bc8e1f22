// tests/emul_serving_records.cc -- TEST INFRASTRUCTURE: the audio history write of microwakeword_b200/csrc/mww_history.h and
// the endpointer records of mww_serving_records.h run on the CPU, unit by unit and row by row as the kernels' threads run
// them, for tests/test_serving_records.py.  Never used by the product.
#include <string.h>

#include "../microwakeword_b200/csrc/mww_serving_records.h"

using namespace mww;

// the write kernel: ring rows ids[i] <- zeros then row i of in, as 8-entry units (the vector form, one 16-byte load of the row or
// zeros, one 16-byte store) when allow_vec and the shape hold, else one entry per unit.  Returns 1 when the vector form ran.
extern "C" int emul_history_write(int16_t *ring, int C, long long seen, const int32_t *ids, int n, int n_samples, const int16_t *in,
                                  long long in_stride, int allow_vec) {
    const HistoryWrite p = history_write_plan(seen, n_samples, C);
    const int vec = allow_vec && history_write_vec_shape(p, in_stride);
    const int units = vec ? C / 8 : C;
    for (long long r = 0; r < n; ++r)
        for (int u = 0; u < units; ++u) {
            int16_t *row = ring + (long long)ids[r] * C;
            const int16_t *src = in + r * in_stride;
            if (vec) {
                const long long t = 8LL * u - p.lead;
                int16_t *dst = row + history_slot(p.slot0, 8 * u, C);
                for (int q = 0; q < 8; ++q) dst[q] = t >= 0 ? src[t + q] : (int16_t)0;
            } else {
                history_write_one(row, src, p, u, C);
            }
        }
    return vec;
}

// out: record_bytes, head, seg, vad, ages, hist
extern "C" void emul_eprec_layout(int vad_window, long long *out) {
    const EpRecLayout L = endpoint_record_layout(vad_window);
    out[0] = L.record_bytes; out[1] = L.head; out[2] = L.seg; out[3] = L.vad; out[4] = L.ages; out[5] = L.hist;
}

namespace {
// cfg: vad_window, n_rows, n_streams; p: hist, seen, flags, armed, elapsed, run, silence, heard, start, speech_end, row_of
EpRecJob job(const int *cfg, long long base, void **p) {
    EpRecJob J;
    J.a.rule = mww_endpoint_rule{cfg[0], 1, 1, 1, 1, 0, 0.5};
    J.a.n_rows = cfg[1]; J.a.n_streams = cfg[2];
    J.a.hist = (float *)p[0]; J.a.seen = (long long *)p[1]; J.a.flags = (unsigned long long *)p[2]; J.a.armed = (int32_t *)p[3];
    J.a.elapsed = (int32_t *)p[4]; J.a.run = (int32_t *)p[5]; J.a.silence = (int32_t *)p[6]; J.a.heard = (int32_t *)p[7];
    J.a.start = (long long *)p[8]; J.a.speech_end = (long long *)p[9]; J.a.row_of = (const int32_t *)p[10];
    J.base = base;
    J.L = endpoint_record_layout(cfg[0]);
    return J;
}
}  // namespace

extern "C" void emul_eprec_pack(const int *cfg, long long base, void **p, const int32_t *ids, int n, uint32_t *rec) {
    const EpRecJob J = job(cfg, base, p);
    for (int i = 0; i < n; ++i) endpoint_record_pack(J, ids[i], rec + (long long)i * (J.L.record_bytes / 4));
}

extern "C" void emul_eprec_unpack(const int *cfg, long long base, void **p, const int32_t *ids, int n, const uint32_t *rec) {
    const EpRecJob J = job(cfg, base, p);
    for (int i = 0; i < n; ++i) endpoint_record_unpack(J, ids[i], rec + (long long)i * (J.L.record_bytes / 4));
}

// the field named by a mismatch, or 0 when the records fit
extern "C" int emul_eprec_mismatch(const mww_endpointer_layout *src, const mww_endpointer_layout *dst, char *name, int cap) {
    const char *f = endpoint_layout_mismatch(*src, *dst);
    if (!f) return 0;
    strncpy(name, f, (size_t)cap - 1);
    name[cap - 1] = 0;
    return 1;
}
