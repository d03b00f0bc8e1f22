// mww_records.cu -- the two kernels of mww_export_streams / mww_import_streams (layout and index math: mww_records.h).
// Pure data movement: each launch moves one part list (the frontend parts, or one model's ring state and pending rows)
// of every listed stream between the handle and the packed records, one word per thread.  A block takes `rpb` whole
// records at a time, so a thread finds its record and word with one 32-bit division; W is the widest word the parts allow.
#include <algorithm>

#include "mww_kernels.h"

namespace mww {

namespace {

constexpr int kRecordThreads = 256;

// handle -> records.  inv: the model's compact index of each global stream id (nullptr: the frontend, indexed by the id).
template <typename W>
__global__ void __launch_bounds__(kRecordThreads)
pack_streams_kernel(RecordJob J, char *__restrict__ rec, long long record_bytes, const int32_t *__restrict__ ids, int n, int rpb, int wpr,
                    RecordBases B, const int32_t *__restrict__ inv) {
    for (long long g = blockIdx.x; g * rpb < n; g += gridDim.x)
        for (int t = threadIdx.x; t < rpb * wpr; t += kRecordThreads) {
            const int jr = t / wpr, w = t - jr * wpr;
            const long long j = g * rpb + jr;
            if (j >= n) break;
            const int id = ids[j];
            record_pack_word<W>(J, w, inv ? inv[id] : id, rec + j * record_bytes, B);
        }
}

// records -> handle; fresh[0, n) (may be nullptr): the members that need the model's fill kernel
template <typename W>
__global__ void __launch_bounds__(kRecordThreads)
unpack_streams_kernel(RecordJob J, const char *__restrict__ rec, long long record_bytes, const int32_t *__restrict__ ids, int n, int rpb,
                      int wpr, RecordBases B, const int32_t *__restrict__ inv, int32_t *__restrict__ fresh) {
    for (long long g = blockIdx.x; g * rpb < n; g += gridDim.x)
        for (int t = threadIdx.x; t < rpb * wpr; t += kRecordThreads) {
            const int jr = t / wpr, w = t - jr * wpr;
            const long long j = g * rpb + jr;
            if (j >= n) break;
            const int id = ids[j];
            record_unpack_word<W>(J, w, inv ? inv[id] : id, rec + j * record_bytes, B, fresh ? fresh + j : nullptr);
        }
}

struct RecordGrid { int rpb, wpr; unsigned blocks; };
RecordGrid record_grid(const RecordJob &J, int word_bytes, int n, int sm_count) {
    RecordGrid G;
    G.wpr = record_words(J, word_bytes);
    G.rpb = std::max(1, kRecordThreads / G.wpr);
    G.blocks = (unsigned)std::max<long long>(1, std::min<long long>(((long long)n + G.rpb - 1) / G.rpb, (long long)sm_count * 8));
    return G;
}

RecordBases record_bases(const void *const *base) {
    RecordBases B;
    for (int p = 0; p < kRecordMaxParts; ++p) B.p[p] = static_cast<char *>(const_cast<void *>(base[p]));
    return B;
}

}  // namespace

cudaError_t launch_pack_streams(const RecordJob &J, void *records, long long record_bytes, const int32_t *ids, int n, const void *const *base,
                                const int32_t *inv, int sm_count, cudaStream_t st) {
    if (n <= 0) return cudaSuccess;
    const int wb = record_word_bytes(J);
    const RecordGrid G = record_grid(J, wb, n, sm_count);
    const RecordBases B = record_bases(base);
    char *rec = static_cast<char *>(records);
    if (wb == 16) pack_streams_kernel<uint4><<<G.blocks, kRecordThreads, 0, st>>>(J, rec, record_bytes, ids, n, G.rpb, G.wpr, B, inv);
    else if (wb == 8) pack_streams_kernel<uint2><<<G.blocks, kRecordThreads, 0, st>>>(J, rec, record_bytes, ids, n, G.rpb, G.wpr, B, inv);
    else if (wb == 4) pack_streams_kernel<uint32_t><<<G.blocks, kRecordThreads, 0, st>>>(J, rec, record_bytes, ids, n, G.rpb, G.wpr, B, inv);
    else pack_streams_kernel<uint8_t><<<G.blocks, kRecordThreads, 0, st>>>(J, rec, record_bytes, ids, n, G.rpb, G.wpr, B, inv);
    return cudaGetLastError();
}

cudaError_t launch_unpack_streams(const RecordJob &J, const void *records, long long record_bytes, const int32_t *ids, int n, void *const *base,
                                  const int32_t *inv, int32_t *fresh, int sm_count, cudaStream_t st) {
    if (n <= 0) return cudaSuccess;
    const int wb = record_word_bytes(J);
    const RecordGrid G = record_grid(J, wb, n, sm_count);
    const RecordBases B = record_bases(base);
    const char *rec = static_cast<const char *>(records);
    if (wb == 16) unpack_streams_kernel<uint4><<<G.blocks, kRecordThreads, 0, st>>>(J, rec, record_bytes, ids, n, G.rpb, G.wpr, B, inv, fresh);
    else if (wb == 8) unpack_streams_kernel<uint2><<<G.blocks, kRecordThreads, 0, st>>>(J, rec, record_bytes, ids, n, G.rpb, G.wpr, B, inv, fresh);
    else if (wb == 4) unpack_streams_kernel<uint32_t><<<G.blocks, kRecordThreads, 0, st>>>(J, rec, record_bytes, ids, n, G.rpb, G.wpr, B, inv, fresh);
    else unpack_streams_kernel<uint8_t><<<G.blocks, kRecordThreads, 0, st>>>(J, rec, record_bytes, ids, n, G.rpb, G.wpr, B, inv, fresh);
    return cudaGetLastError();
}

}  // namespace mww
