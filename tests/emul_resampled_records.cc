// tests/emul_resampled_records.cc -- TEST INFRASTRUCTURE: the resampler part of a resampled stream record
// (mww_export_resampled_streams) through the record emulation of tests/emul_records.cc, for tests/test_resampled_records.py.
// The job is the one the C-ABI builds (record_job_resampler of microwakeword_b200/csrc/mww_records.h), moved word by word
// with the pack / unpack bodies the kernels run.
#include <stddef.h>

#include "emul_records.cc"

// out[0..6) = n_parts, bytes[0], padded[0], rec_off[0], the word size the kernels move it with, words per record
extern "C" void emul_resampler_job_shape(long long rec_off, int hist_stride, long long *out) {
    const RecordJob J = record_job_resampler(rec_off, hist_stride);
    const int wb = record_word_bytes(J);
    out[0] = J.n_parts; out[1] = J.bytes[0]; out[2] = J.padded[0]; out[3] = J.rec_off[0]; out[4] = wb; out[5] = record_words(J, wb);
}

// export (pack != 0) or import of the resampler part of n records `record_bytes` apart, for streams ids of a history
// [n_streams][hist_stride] int16.  Returns the word size.
extern "C" int emul_resampler_job(int pack, long long rec_off, int hist_stride, char *rec, long long record_bytes, const int32_t *ids, int n,
                                  char *hist) {
    const RecordJob J = record_job_resampler(rec_off, hist_stride);
    const RecordBases B{{hist, nullptr, nullptr}};
    const int wb = record_word_bytes(J);
    if (wb == 16) move<Word16>(pack, J, rec, record_bytes, ids, n, B, nullptr, nullptr);
    else if (wb == 8) move<Word8>(pack, J, rec, record_bytes, ids, n, B, nullptr, nullptr);
    else if (wb == 4) move<uint32_t>(pack, J, rec, record_bytes, ids, n, B, nullptr, nullptr);
    else move<uint8_t>(pack, J, rec, record_bytes, ids, n, B, nullptr, nullptr);
    return wb;
}

extern "C" int emul_resampler_part_samples() { return kRecordResamplerSamples; }

// sizeof, then the offsets of record_bytes, resampler_off, rate, reserved, inputs_seen, samples16_seen
extern "C" void emul_resampler_layout_offsets(long long *out) {
    out[0] = sizeof(mww_resampler_layout);
    out[1] = offsetof(mww_resampler_layout, record_bytes); out[2] = offsetof(mww_resampler_layout, resampler_off);
    out[3] = offsetof(mww_resampler_layout, rate); out[4] = offsetof(mww_resampler_layout, reserved);
    out[5] = offsetof(mww_resampler_layout, inputs_seen); out[6] = offsetof(mww_resampler_layout, samples16_seen);
}
