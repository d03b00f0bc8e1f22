// mww_detector_records.cu -- the two kernels of mww_export_detector_rows / mww_import_detector_rows (layout and per-word
// bodies: mww_detector_records.h).  Pure data movement: one launch moves every used model's slot of every listed record,
// one 4-byte word per thread, with the model descriptors in a __grid_constant__ parameter, so the launch count does not
// depend on n or on the model count.  A block takes `rpb` whole records at a time, so a thread finds its record and word
// with one 32-bit division.  A companion library of its own, libmww_detector_records.so, so that libmww_b200.so and the
// three detector libraries keep exactly the kernels they had.
#include <algorithm>

#include "mww_kernels.h"

namespace mww {

namespace {

constexpr int kDetRecThreads = 256;

// detector -> records [n][J.words]
__global__ void __launch_bounds__(kDetRecThreads)
pack_detector_rows_kernel(const __grid_constant__ DetRecJob J, uint32_t *__restrict__ rec, const int32_t *__restrict__ ids, int n, int rpb) {
    const int wpr = J.words;
    for (long long g = blockIdx.x; g * rpb < n; g += gridDim.x)
        for (int t = threadIdx.x; t < rpb * wpr; t += kDetRecThreads) {
            const int jr = t / wpr, w = t - jr * wpr;
            const long long j = g * rpb + jr;
            if (j >= n) break;
            detector_record_pack_word(J, w, ids[j], rec + j * wpr);
        }
}

// records [n][J.words] -> detector
__global__ void __launch_bounds__(kDetRecThreads)
unpack_detector_rows_kernel(const __grid_constant__ DetRecJob J, const uint32_t *__restrict__ rec, const int32_t *__restrict__ ids, int n, int rpb) {
    const int wpr = J.words;
    for (long long g = blockIdx.x; g * rpb < n; g += gridDim.x)
        for (int t = threadIdx.x; t < rpb * wpr; t += kDetRecThreads) {
            const int jr = t / wpr, w = t - jr * wpr;
            const long long j = g * rpb + jr;
            if (j >= n) break;
            detector_record_unpack_word(J, w, ids[j], rec + j * wpr);
        }
}

struct DetRecGrid { int rpb; unsigned blocks; };
DetRecGrid detector_record_grid(const DetRecJob &J, int n) {
    DetRecGrid G;
    G.rpb = std::max(1, kDetRecThreads / J.words);
    G.blocks = (unsigned)std::max<long long>(1, std::min<long long>(((long long)n + G.rpb - 1) / G.rpb, 4096));
    return G;
}

}  // namespace

cudaError_t launch_pack_detector_rows(const DetRecJob &J, void *records, const int32_t *ids, int n, cudaStream_t st) {
    if (n <= 0) return cudaSuccess;
    const DetRecGrid G = detector_record_grid(J, n);
    pack_detector_rows_kernel<<<G.blocks, kDetRecThreads, 0, st>>>(J, static_cast<uint32_t *>(records), ids, n, G.rpb);
    return cudaGetLastError();
}

cudaError_t launch_unpack_detector_rows(const DetRecJob &J, const void *records, const int32_t *ids, int n, cudaStream_t st) {
    if (n <= 0) return cudaSuccess;
    const DetRecGrid G = detector_record_grid(J, n);
    unpack_detector_rows_kernel<<<G.blocks, kDetRecThreads, 0, st>>>(J, static_cast<const uint32_t *>(records), ids, n, G.rpb);
    return cudaGetLastError();
}

}  // namespace mww
