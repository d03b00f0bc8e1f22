// tests/emul_records.cc -- TEST INFRASTRUCTURE: the record layout, the per-word bodies of the pack / unpack kernels and the
// layout comparison of microwakeword_b200/csrc/mww_records.h run on the CPU, for tests/test_stream_records.py.
#include <string.h>

#include "../microwakeword_b200/csrc/mww_records.h"

using namespace mww;

namespace {
struct alignas(16) Word16 { uint64_t a, b; };
struct alignas(8) Word8 { uint64_t a; };

RecordLayout layout_of(const long long *state_bytes, const long long *pend_bytes, int n_models) {
    RecordModel rm[kRecordMaxModels];
    for (int k = 0; k < n_models; ++k) rm[k] = RecordModel{state_bytes[k], pend_bytes[k]};
    return record_layout(rm, n_models);
}

template <typename W>
void move(bool pack, const RecordJob &J, char *rec, long long record_bytes, const int32_t *ids, int n, const RecordBases &B, const int32_t *inv,
          int32_t *fresh) {
    const int wpr = record_words(J, (int)sizeof(W));
    for (int j = 0; j < n; ++j)
        for (int w = 0; w < wpr; ++w) {
            const int c = inv ? inv[ids[j]] : ids[j];
            if (pack) record_pack_word<W>(J, w, c, rec + j * record_bytes, B);
            else record_unpack_word<W>(J, w, c, rec + j * record_bytes, B, fresh ? fresh + j : nullptr);
        }
}
}  // namespace

// out[0..3) = record_bytes, carry_off, estimate_off; then nn_off[n_models], pend_off[n_models]
extern "C" void emul_record_layout(const long long *state_bytes, const long long *pend_bytes, int n_models, long long *out) {
    const RecordLayout L = layout_of(state_bytes, pend_bytes, n_models);
    out[0] = L.record_bytes; out[1] = L.carry_off; out[2] = L.estimate_off;
    for (int k = 0; k < n_models; ++k) { out[3 + k] = L.nn_off[k]; out[3 + n_models + k] = L.pend_off[k]; }
}

// One job of an export (pack != 0) or import over host buffers, word by word as the kernels run it: model k's state and
// pending rows with the given rotating rings, or the frontend parts for k < 0 (base0 unused, base1 carry, base2 estimate).
// Returns the word size the job moves with.
extern "C" int emul_record_job(int pack, int k, const long long *state_bytes, const long long *pend_bytes, int n_models, int n_rings,
                               const int *ring_off, const int *ring_row_bytes, const int *ring_rows, const int *heads, char *rec,
                               const int32_t *ids, int n, char *base0, char *base1, char *base2, const int32_t *inv, int32_t *fresh, int zero_fresh) {
    const RecordLayout L = layout_of(state_bytes, pend_bytes, n_models);
    RecordJob J = k < 0 ? record_job_frontend(L) : record_job_model(L, k, RecordModel{state_bytes[k], pend_bytes[k]});
    J.zero_fresh = zero_fresh != 0;
    for (int i = 0; i < n_rings; ++i) record_add_ring(&J, ring_off[i], ring_row_bytes[i], ring_rows[i], heads[i]);
    const RecordBases B{{base0, base1, base2}};
    const int wb = record_word_bytes(J);
    if (wb == 16) move<Word16>(pack, J, rec, L.record_bytes, ids, n, B, inv, fresh);
    else if (wb == 8) move<Word8>(pack, J, rec, L.record_bytes, ids, n, B, inv, fresh);
    else if (wb == 4) move<uint32_t>(pack, J, rec, L.record_bytes, ids, n, B, inv, fresh);
    else move<uint8_t>(pack, J, rec, L.record_bytes, ids, n, B, inv, fresh);
    return wb;
}

extern "C" int emul_sizeof_stream_layout() { return (int)sizeof(mww_stream_layout); }

// field_out: the name of the first differing field ("" when the layouts fit); returns the model index or -1
extern "C" int emul_layout_mismatch(const mww_stream_layout *src, const mww_stream_layout *dst, char *field_out) {
    int index = -1;
    const char *f = stream_layout_mismatch(*src, *dst, &index);
    strcpy(field_out, f ? f : "");
    return index;
}

extern "C" uint64_t emul_record_model_hash(uint64_t container_hash, int quantized, long long state_elems) {
    return record_model_hash(container_hash, quantized != 0, state_elems);
}
