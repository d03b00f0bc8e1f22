// mww_serving_records.cu -- the kernels that let a stream's serving state move with it between handles: the audio history
// write (mww_write_audio_history; index math in mww_history.h) and the pack and unpack of endpointer records
// (mww_export_endpointer_rows / mww_import_endpointer_rows; layout and per-row bodies in mww_serving_records.h).  Pure data
// movement, one launch per call whatever n is.  The history write moves 8-sample units over rows x units in a grid-stride
// loop, as the append and read kernels do; the record kernels run a thread per listed id with the endpointer's state and
// layout in a __grid_constant__ parameter.  A companion library of its own, libmww_serving_records.so, so that
// libmww_b200.so, libmww_history.so and libmww_endpoint.so keep exactly the kernels they had.
#include <algorithm>

#include "mww_kernels.h"

namespace mww {

namespace {

constexpr int kServingThreads = 256;

// ring rows ids[i] <- zeros followed by row i of `in` (history_write_one); vec: units of 8 entries, 16-byte loads and stores
__global__ void __launch_bounds__(kServingThreads)
history_write_kernel(int16_t *__restrict__ ring, int C, const int32_t *__restrict__ ids, int n, HistoryWrite p, const int16_t *__restrict__ in,
                     long long in_stride, int vec) {
    const int units = vec ? C / 8 : C;
    const long long total = (long long)n * units;
    for (long long i = (long long)blockIdx.x * kServingThreads + threadIdx.x; i < total; i += (long long)gridDim.x * kServingThreads) {
        const long long r = i / units;
        const int u = (int)(i - r * units);
        int16_t *row = ring + (long long)ids[r] * C;
        const int16_t *src = in + r * in_stride;
        if (vec) {
            const long long t = 8LL * u - p.lead;
            const uint4 v = t >= 0 ? *reinterpret_cast<const uint4 *>(src + t) : make_uint4(0, 0, 0, 0);
            *reinterpret_cast<uint4 *>(row + history_slot(p.slot0, 8 * u, C)) = v;
        } else {
            history_write_one(row, src, p, u, C);
        }
    }
}

// endpointer -> records [n][record_bytes], a thread per listed id
__global__ void __launch_bounds__(kServingThreads)
pack_endpointer_rows_kernel(const __grid_constant__ EpRecJob J, uint32_t *__restrict__ rec, const int32_t *__restrict__ ids, int n) {
    const int i = blockIdx.x * kServingThreads + threadIdx.x;
    if (i < n) endpoint_record_pack(J, ids[i], rec + (long long)i * (J.L.record_bytes / 4));
}

// records [n][record_bytes] -> endpointer
__global__ void __launch_bounds__(kServingThreads)
unpack_endpointer_rows_kernel(const __grid_constant__ EpRecJob J, const uint32_t *__restrict__ rec, const int32_t *__restrict__ ids, int n) {
    const int i = blockIdx.x * kServingThreads + threadIdx.x;
    if (i < n) endpoint_record_unpack(J, ids[i], rec + (long long)i * (J.L.record_bytes / 4));
}

unsigned serving_blocks(long long total) { return (unsigned)std::max<long long>(1, (total + kServingThreads - 1) / kServingThreads); }

}  // namespace

// The vector form applies when history_write_vec_shape holds and `in` is 16-byte aligned.  Rows of the ring start on 16 bytes
// (C % 8 == 0, cudaMalloc alignment).
cudaError_t launch_history_write(int16_t *ring, int C, long long seen, const int32_t *ids, int n, int n_samples, const int16_t *in,
                                 long long in_stride, int sm_count, cudaStream_t st) {
    if (n <= 0 || C <= 0) return cudaSuccess;
    const HistoryWrite p = history_write_plan(seen, n_samples, C);
    const int vec = history_write_vec_shape(p, in_stride) && reinterpret_cast<uintptr_t>(in) % 16 == 0;
    const long long total = (long long)n * (vec ? C / 8 : C);
    const unsigned blocks = (unsigned)std::min<long long>(serving_blocks(total), (long long)sm_count * 16);
    history_write_kernel<<<blocks, kServingThreads, 0, st>>>(ring, C, ids, n, p, in, in_stride, vec);
    return cudaGetLastError();
}

cudaError_t launch_pack_endpointer_rows(const EpRecJob &J, void *records, const int32_t *ids, int n, cudaStream_t st) {
    if (n <= 0) return cudaSuccess;
    pack_endpointer_rows_kernel<<<serving_blocks(n), kServingThreads, 0, st>>>(J, static_cast<uint32_t *>(records), ids, n);
    return cudaGetLastError();
}

cudaError_t launch_unpack_endpointer_rows(const EpRecJob &J, const void *records, const int32_t *ids, int n, cudaStream_t st) {
    if (n <= 0) return cudaSuccess;
    unpack_endpointer_rows_kernel<<<serving_blocks(n), kServingThreads, 0, st>>>(J, static_cast<const uint32_t *>(records), ids, n);
    return cudaGetLastError();
}

}  // namespace mww
