// mww_streams.cu -- the three small kernels of per-model stream sets (index math: mww_streams.h).  None of them touches an
// NN or frontend kernel: a model on a subset of the streams runs the usual kernels on compact state and compact rows.
#include <algorithm>

#include "mww_kernels.h"
#include "mww_streams.h"

namespace mww {

namespace {

unsigned grid_for(long long total, int sm_count) {
    return (unsigned)std::max<long long>(1, std::min<long long>((total + 255) / 256, (long long)sm_count * 16));
}

// feature rows of a tile's members -> compact [m][F][40] rows; a stream's F x 80 bytes are contiguous and 16-byte aligned
__global__ void gather_rows_kernel(const uint4 *__restrict__ feat, const int32_t *__restrict__ ids, int a, int first,
                                   long long chunks_per_stream, long long total, uint4 *__restrict__ out) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
        out[i] = feat[gather_source(i, chunks_per_stream, ids, a, first)];
}

template <typename W>
__global__ void remap_rows_kernel(W *__restrict__ dst, const W *__restrict__ src, long long words_per_row, const int32_t *__restrict__ old_index,
                                  long long total) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long s = remap_source(i, words_per_row, old_index);
        if (s >= 0) dst[i] = src[s];
    }
}

__global__ void compact_ids_kernel(int32_t *__restrict__ out, const int32_t *__restrict__ ids, int n, const int32_t *__restrict__ inv,
                                   int n_streams) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) out[i] = compact_id(ids[i], inv, n_streams);
}

}  // namespace

cudaError_t launch_gather_rows(const uint16_t *feat, const int32_t *ids, int a, int first, int m, int n_rows, uint16_t *out, int sm_count,
                               cudaStream_t st) {
    const long long chunks = (long long)n_rows * kNumChannels * 2 / 16;
    const long long total = (long long)m * chunks;
    if (total <= 0) return cudaSuccess;
    gather_rows_kernel<<<grid_for(total, sm_count), 256, 0, st>>>(reinterpret_cast<const uint4 *>(feat), ids, a, first, chunks, total,
                                                                   reinterpret_cast<uint4 *>(out));
    return cudaGetLastError();
}

cudaError_t launch_remap_rows(void *dst, const void *src, size_t bytes_per_row, const int32_t *old_index, int n_new, int sm_count,
                              cudaStream_t st) {
    if (n_new <= 0 || bytes_per_row == 0) return cudaSuccess;
    if (bytes_per_row % 4 == 0) {
        const long long words = (long long)(bytes_per_row / 4), total = words * n_new;
        remap_rows_kernel<<<grid_for(total, sm_count), 256, 0, st>>>(static_cast<uint32_t *>(dst), static_cast<const uint32_t *>(src), words,
                                                                      old_index, total);
    } else {
        const long long total = (long long)bytes_per_row * n_new;
        remap_rows_kernel<<<grid_for(total, sm_count), 256, 0, st>>>(static_cast<uint8_t *>(dst), static_cast<const uint8_t *>(src),
                                                                      (long long)bytes_per_row, old_index, total);
    }
    return cudaGetLastError();
}

cudaError_t launch_compact_ids(int32_t *out, const int32_t *ids, int n, const int32_t *inv, int n_streams, int sm_count, cudaStream_t st) {
    if (n <= 0) return cudaSuccess;
    compact_ids_kernel<<<grid_for(n, sm_count), 256, 0, st>>>(out, ids, n, inv, n_streams);
    return cudaGetLastError();
}

}  // namespace mww
