// mww_records.h -- the packed stream record of mww_export_streams / mww_import_streams and the index math of the two
// kernels that fill and read it (mww_records.cu).  One record holds everything one stream of a handle carries:
//
//     uint64  member_mask                  bit k: the stream was a member of model k and slot k holds its state
//     int16   carry[480]                   window buffer
//     uint32  estimate[40]                 noise estimates
//     for each model k of the handle:      nn[state bytes]     rings CANONICAL (oldest row first), as mww_get_model_state
//                                          pending[pend bytes] the model's pending-row buffer
//
// every part padded to 16 bytes.  record_layout() is the only place that knows the offsets.  The kernels move one PART LIST
// (RecordJob) per launch -- the frontend parts, or one model's two -- a word at a time; record_word() says where word w of
// a record lives in the record and in the handle, with the rows of a rotated ring (okay_nabu live calls, LiveHeads) mapped
// to the physical row that holds them.  CUDA-free apart from MWW_HD, so that tests/emul_records.cc runs the same functions
// on the CPU.
#pragma once

#include "../../include/mww.h"
#include "mww_common.h"

namespace mww {

constexpr int kRecordMaxModels = 64;          // one 64-bit member mask
constexpr int kRecordMaxParts = 3;
constexpr int kRecordMaxRings = 5;

inline long long record_pad16(long long bytes) { return (bytes + 15) / 16 * 16; }

// what the layout needs to know of a model: bytes per stream of its ring state and of its pending-row buffer
struct RecordModel { long long state_bytes, pend_bytes; };

struct RecordLayout {
    long long record_bytes, carry_off, estimate_off;
    long long nn_off[kRecordMaxModels], pend_off[kRecordMaxModels];
};

inline RecordLayout record_layout(const RecordModel *models, int n_models) {
    RecordLayout L{};
    long long off = record_pad16(sizeof(uint64_t));
    L.carry_off = off;
    off += record_pad16(kWindow * sizeof(int16_t));
    L.estimate_off = off;
    off += record_pad16(kNumChannels * sizeof(uint32_t));
    for (int k = 0; k < n_models; ++k) {
        L.nn_off[k] = off;
        off += record_pad16(models[k].state_bytes);
        L.pend_off[k] = off;
        off += record_pad16(models[k].pend_bytes);
    }
    L.record_bytes = off;
    return L;
}

// a rotating ring inside part 0 of a job: `rows` rows of 1 << row_shift bytes from byte `off` of the stream's state;
// logical row r (0 = oldest) is physical row (head + r) % rows
struct RecordRing { int off, row_shift, rows, head; };

// the parts one launch moves for every listed stream.  Part p is bytes[p] bytes per stream in the handle (streams packed
// at that pitch) and padded[p] >= bytes[p] bytes at rec_off[p] of the record.
struct RecordJob {
    int n_parts = 0;
    long long rec_off[kRecordMaxParts] = {0, 0, 0};
    int bytes[kRecordMaxParts] = {0, 0, 0}, padded[kRecordMaxParts] = {0, 0, 0};
    int n_rings = 0;
    RecordRing ring[kRecordMaxRings] = {};
    int model_bit = -1;         // bit of the member mask this job's model owns; -1: the frontend parts
    bool zero_fresh = false;    // the model's fresh state is all zero bytes (fp32, hybrid): import writes it itself
};

inline void record_add_part(RecordJob *J, long long rec_off, long long bytes) {
    J->rec_off[J->n_parts] = rec_off;
    J->bytes[J->n_parts] = (int)bytes;
    J->padded[J->n_parts] = (int)record_pad16(bytes);
    J->n_parts += 1;
}
// row_bytes must be a power of two (okay_nabu's rings: 32 or 64 channels of 1 or 4 bytes)
inline void record_add_ring(RecordJob *J, int off, int row_bytes, int rows, int head) {
    int shift = 0;
    while ((1 << shift) < row_bytes) ++shift;
    J->ring[J->n_rings++] = RecordRing{off, shift, rows, head};
}

// mask word (zero on export: the model jobs set their bits afterwards), window carry, noise estimates
inline RecordJob record_job_frontend(const RecordLayout &L) {
    RecordJob J;
    record_add_part(&J, 0, 0);
    J.padded[0] = (int)L.carry_off;          // the mask word and its padding: nothing of the handle, all of it zeroed
    record_add_part(&J, L.carry_off, kWindow * sizeof(int16_t));
    record_add_part(&J, L.estimate_off, kNumChannels * sizeof(uint32_t));
    return J;
}
// model k's ring state (part 0; add its rotating rings with record_add_ring) and pending rows
inline RecordJob record_job_model(const RecordLayout &L, int k, const RecordModel &m) {
    RecordJob J;
    record_add_part(&J, L.nn_off[k], m.state_bytes);
    record_add_part(&J, L.pend_off[k], m.pend_bytes);
    J.model_bit = k;
    return J;
}

// The resampler part of a resampled record (mww_export_resampled_streams), at rec_off = the stream record's record_bytes:
// int16 hist[kRecordResamplerSamples], the first hist_stride samples of the stream's history row, zeros after them.  One
// plain span per stream at the handle's row pitch (0 at 16 kHz: the whole part is padding, written as zero).
constexpr int kRecordResamplerSamples = 244;        // the per-stream-rate row: H_max = 243 rounded up to even
constexpr int kRecordResamplerBytes = kRecordResamplerSamples * 2;
constexpr int kRecordResamplerPart = 496;           // kRecordResamplerBytes padded to 16

inline RecordJob record_job_resampler(long long rec_off, int hist_stride) {
    RecordJob J;
    record_add_part(&J, rec_off, (long long)hist_stride * 2);
    J.padded[0] = kRecordResamplerPart;
    return J;
}

// widest word (16, 8, 4 or 1 bytes) that divides every part and every ring's offset and row, so that no word straddles a
// part, a stream or a ring row: 16 for the frontend and for okay_nabu, fp32 (rows of 128 / 256 bytes) and int8 (32 / 64)
// alike; whatever the span allows for a run-time geometry
inline int record_word_bytes(const RecordJob &J) {
    for (int w = 16; w >= 4; w >>= 1) {
        bool ok = true;
        for (int p = 0; p < J.n_parts; ++p) ok = ok && J.bytes[p] % w == 0;
        for (int i = 0; i < J.n_rings; ++i) ok = ok && J.ring[i].off % w == 0 && (1 << J.ring[i].row_shift) % w == 0;
        if (ok) return w;
    }
    return 1;
}
inline int record_words(const RecordJob &J, int word_bytes) {
    int b = 0;
    for (int p = 0; p < J.n_parts; ++p) b += J.padded[p];
    return b / word_bytes;
}

// byte offset inside a stream's state of canonical byte `b` of part 0, under the job's ring rotation
MWW_HD int record_rotated(const RecordJob &J, int b) {
    for (int i = 0; i < kRecordMaxRings; ++i) {
        if (i >= J.n_rings) break;
        const RecordRing g = J.ring[i];
        const int rel = b - g.off;
        if (rel < 0 || rel >= (g.rows << g.row_shift)) continue;
        const int r = rel >> g.row_shift;
        int p = g.head + r;
        if (p >= g.rows) p -= g.rows;
        return b + ((p - r) << g.row_shift);
    }
    return b;
}

// word w of a record's share of job J: part, byte offset in the record, byte offset in the stream's part of the handle
// (-1: padding, which export writes as zero and import skips)
struct RecordWord { int part; long long rec_off; int state_off; };
MWW_HD RecordWord record_word(const RecordJob &J, int w, int word_bytes) {
    int b = w * word_bytes, part = 0;
    for (int p = 0; p + 1 < kRecordMaxParts; ++p)
        if (p + 1 < J.n_parts && part == p && b >= J.padded[p]) { b -= J.padded[p]; part = p + 1; }
    RecordWord r;
    r.part = part;
    r.rec_off = J.rec_off[part] + b;
    r.state_off = b >= J.bytes[part] ? -1 : (part == 0 ? record_rotated(J, b) : b);
    return r;
}

// The body of the two kernels, one word of one record (W: a 16-, 8-, 4- or 1-byte word type).  B.p[p]: part p of stream /
// compact index 0 in the handle; c: the stream's index there, -1 when it is not a member of the job's model.
struct RecordBases { char *p[kRecordMaxParts]; };
MWW_HD char *record_part_base(const RecordBases &B, int part) { return part == 0 ? B.p[0] : (part == 1 ? B.p[1] : B.p[2]); }

// handle -> record.  Padding and the slots of non-members are written as zero; a member sets its model's bit of the mask
// word, which the frontend job of the same call zeroed before.
template <typename W>
MWW_HD void record_pack_word(const RecordJob &J, int w, int c, char *rec, const RecordBases &B) {
    const RecordWord rw = record_word(J, w, (int)sizeof(W));
    W v{};
    if (c >= 0 && rw.state_off >= 0)
        v = *reinterpret_cast<const W *>(record_part_base(B, rw.part) + (long long)c * J.bytes[rw.part] + rw.state_off);
    *reinterpret_cast<W *>(rec + rw.rec_off) = v;
    if (w == 0 && J.model_bit >= 0 && c >= 0) *reinterpret_cast<unsigned long long *>(rec) |= 1ull << J.model_bit;
}

// record -> handle, for a member whose mask bit is set.  A member whose bit is clear starts fresh: zeros written here when
// that is the model's fresh state, else *fresh (when given) = c and the caller runs the model's fill kernel over the list;
// *fresh = -1 for every other record.
template <typename W>
MWW_HD void record_unpack_word(const RecordJob &J, int w, int c, const char *rec, const RecordBases &B, int32_t *fresh) {
    const RecordWord rw = record_word(J, w, (int)sizeof(W));
    if (c < 0 && !(w == 0 && fresh)) return;
    bool has = true;
    if (J.model_bit >= 0) has = (*reinterpret_cast<const unsigned long long *>(rec) >> J.model_bit) & 1ull;
    if (w == 0 && fresh) *fresh = c >= 0 && !has ? c : -1;
    if (c < 0 || rw.state_off < 0 || (!has && !J.zero_fresh)) return;
    W v{};
    if (has) v = *reinterpret_cast<const W *>(rec + rw.rec_off);
    *reinterpret_cast<W *>(record_part_base(B, rw.part) + (long long)c * J.bytes[rw.part] + rw.state_off) = v;
}

// The first field in which the layout the records were exported with differs from the importing handle's own, nullptr
// when the records fit.  *index = the model concerned for a per-model field, else -1.  rows_are_features is not compared:
// it travels with the records and only lowers the destination's flag.
inline const char *stream_layout_mismatch(const mww_stream_layout &src, const mww_stream_layout &dst, int *index) {
    *index = -1;
    if (src.n_models != dst.n_models) return "n_models";
    for (int k = 0; k < dst.n_models && k < kRecordMaxModels; ++k)
        if (src.model_hash[k] != dst.model_hash[k]) { *index = k; return "model_hash"; }
    if (src.record_bytes != dst.record_bytes) return "record_bytes";
    if (src.hop_samples != dst.hop_samples) return "hop_samples";
    if (src.frontend_buffered != dst.frontend_buffered) return "frontend_buffered";
    for (int k = 0; k < dst.n_models && k < kRecordMaxModels; ++k)
        if (src.pending_rows[k] != dst.pending_rows[k]) { *index = k; return "pending_rows"; }
    return nullptr;
}

// the model identity a layout carries: the container's hash with the precision and ring-state size folded in
inline uint64_t record_model_hash(uint64_t container_hash, bool quantized, long long state_elems) {
    uint64_t x = container_hash;
    x = (x ^ (uint64_t)(quantized ? 1 : 0)) * 1099511628211ull;
    x = (x ^ (uint64_t)state_elems) * 1099511628211ull;
    return x;
}

}  // namespace mww
