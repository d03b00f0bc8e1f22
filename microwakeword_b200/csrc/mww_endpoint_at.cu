// mww_endpoint_at.cu -- the positioned forms of the endpointer's kernels (rule in include/mww.h, "positioned arm"; per-row
// bodies in mww_endpoint.h and mww_serving_records.h, instantiated with kAt = true): the update that mutes the steps within an
// arm_at's skip, the arm and the clear that zero the mute word, the two passes of arm_at (the reduction of each row's latest
// position, then the arm) and the record pack and unpack that carry the mute word.  An endpointer runs these for good from its
// first arm_at, set_mutes or import of positioned records, and the plain kernels before.  A thread per row or listed id, the
// rule and state pointers in __grid_constant__ parameters as in mww_endpoint.cu.  A companion library of its own,
// libmww_endpoint_at.so, so that libmww_endpoint.so and libmww_serving_records.so keep exactly the kernels they had.
#include <algorithm>

#include "mww_kernels.h"

namespace mww {

namespace {

constexpr int kEndpointAtThreads = 256;

__global__ void __launch_bounds__(kEndpointAtThreads)
endpoint_update_muted_kernel(const __grid_constant__ EndpointArgs a, int32_t *__restrict__ mute, const float *__restrict__ probs, long long pitch,
                             int n, long long pos0) {
    const int r = blockIdx.x * kEndpointAtThreads + threadIdx.x;
    if (r < a.n_rows) endpoint_update_row_t<true>(a, mute, r, probs, pitch, n, pos0);
}

__global__ void __launch_bounds__(kEndpointAtThreads)
endpoint_arm_muted_kernel(const __grid_constant__ EndpointArgs a, const __grid_constant__ EndpointReplay R, int32_t *__restrict__ mute,
                          const int32_t *__restrict__ ids, int n) {
    const int i = blockIdx.x * kEndpointAtThreads + threadIdx.x;
    if (i < n) endpoint_arm_one_t<true>(a, mute, R, ids[i]);
}

// ids == nullptr: rows [0, n_rows); else the rows of the n listed global ids (ids outside the set ignored)
__global__ void __launch_bounds__(kEndpointAtThreads)
endpoint_clear_muted_kernel(const __grid_constant__ EndpointArgs a, int32_t *__restrict__ mute, const int32_t *__restrict__ ids, int n, int reset) {
    const int i = blockIdx.x * kEndpointAtThreads + threadIdx.x;
    if (i >= n) return;
    const int r = ids ? endpoint_row(a, ids[i]) : i;
    if (r >= 0) endpoint_clear_row_t<true>(a, mute, r, reset);
}

__global__ void __launch_bounds__(kEndpointAtThreads)
endpoint_at_reduce_kernel(const __grid_constant__ EndpointArgs a, const __grid_constant__ EndpointAt A, const int32_t *__restrict__ ids,
                          const long long *__restrict__ positions, int n) {
    const int i = blockIdx.x * kEndpointAtThreads + threadIdx.x;
    if (i < n) endpoint_at_reduce_one(a, A, ids[i], positions[i]);
}

__global__ void __launch_bounds__(kEndpointAtThreads)
endpoint_arm_at_kernel(const __grid_constant__ EndpointArgs a, const __grid_constant__ EndpointAt A, const int32_t *__restrict__ ids,
                       const long long *__restrict__ positions, int n) {
    const int i = blockIdx.x * kEndpointAtThreads + threadIdx.x;
    if (i < n) endpoint_arm_at_one(a, A, ids[i], positions[i]);
}

__global__ void __launch_bounds__(kEndpointAtThreads)
pack_endpointer_rows_muted_kernel(const __grid_constant__ EpRecJob J, const int32_t *__restrict__ mute, uint32_t *__restrict__ rec,
                                  const int32_t *__restrict__ ids, int n) {
    const int i = blockIdx.x * kEndpointAtThreads + threadIdx.x;
    if (i < n) endpoint_record_pack_t<true>(J, mute, ids[i], rec + (long long)i * (J.L.record_bytes / 4));
}

__global__ void __launch_bounds__(kEndpointAtThreads)
unpack_endpointer_rows_muted_kernel(const __grid_constant__ EpRecJob J, int32_t *__restrict__ mute, const uint32_t *__restrict__ rec,
                                    const int32_t *__restrict__ ids, int n) {
    const int i = blockIdx.x * kEndpointAtThreads + threadIdx.x;
    if (i < n) endpoint_record_unpack_t<true>(J, mute, ids[i], rec + (long long)i * (J.L.record_bytes / 4));
}

unsigned endpoint_at_blocks(long long n) { return (unsigned)std::max<long long>(1, (n + kEndpointAtThreads - 1) / kEndpointAtThreads); }

}  // namespace

cudaError_t launch_endpoint_update_muted(const EndpointArgs &a, int32_t *mute, const float *probs, long long pitch, int n, long long pos0,
                                         cudaStream_t st) {
    endpoint_update_muted_kernel<<<endpoint_at_blocks(a.n_rows), kEndpointAtThreads, 0, st>>>(a, mute, probs, pitch, n, pos0);
    return cudaGetLastError();
}

cudaError_t launch_endpoint_arm_muted(const EndpointArgs &a, const EndpointReplay &R, int32_t *mute, const int32_t *ids, int n, cudaStream_t st) {
    endpoint_arm_muted_kernel<<<endpoint_at_blocks(n), kEndpointAtThreads, 0, st>>>(a, R, mute, ids, n);
    return cudaGetLastError();
}

cudaError_t launch_endpoint_clear_muted(const EndpointArgs &a, int32_t *mute, const int32_t *ids, int n, int reset, cudaStream_t st) {
    endpoint_clear_muted_kernel<<<endpoint_at_blocks(n), kEndpointAtThreads, 0, st>>>(a, mute, ids, n, reset);
    return cudaGetLastError();
}

cudaError_t launch_endpoint_arm_at(const EndpointArgs &a, const EndpointAt &A, const int32_t *ids, const long long *positions, int n,
                                   cudaStream_t st) {
    endpoint_at_reduce_kernel<<<endpoint_at_blocks(n), kEndpointAtThreads, 0, st>>>(a, A, ids, positions, n);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    endpoint_arm_at_kernel<<<endpoint_at_blocks(n), kEndpointAtThreads, 0, st>>>(a, A, ids, positions, n);
    return cudaGetLastError();
}

cudaError_t launch_pack_endpointer_rows_muted(const EpRecJob &J, const int32_t *mute, void *records, const int32_t *ids, int n, cudaStream_t st) {
    if (n <= 0) return cudaSuccess;
    pack_endpointer_rows_muted_kernel<<<endpoint_at_blocks(n), kEndpointAtThreads, 0, st>>>(J, mute, static_cast<uint32_t *>(records), ids, n);
    return cudaGetLastError();
}

cudaError_t launch_unpack_endpointer_rows_muted(const EpRecJob &J, int32_t *mute, const void *records, const int32_t *ids, int n,
                                                cudaStream_t st) {
    if (n <= 0) return cudaSuccess;
    unpack_endpointer_rows_muted_kernel<<<endpoint_at_blocks(n), kEndpointAtThreads, 0, st>>>(J, mute, static_cast<const uint32_t *>(records),
                                                                                             ids, n);
    return cudaGetLastError();
}

}  // namespace mww
