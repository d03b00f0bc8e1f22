// mww_endpoint.cu -- the four kernels of the endpointer (rule in include/mww.h, per-row bodies in mww_endpoint.h): the update
// (a thread per row, steps walked in order), the arm with its replay and the reset / disarm (a thread per listed id or row),
// and the command read (8-sample units over event slots x samples in a grid-stride loop, as the history read).  The rule and
// the state pointers travel in a __grid_constant__ EndpointArgs, the replay positions in a __grid_constant__ EndpointReplay,
// so that no kernel copies them to local memory.  A companion library of its own, libmww_endpoint.so, so that
// libmww_b200.so and the other companion libraries keep exactly the kernels they had.
#include <algorithm>

#include "mww_kernels.h"

namespace mww {

namespace {

constexpr int kEndpointThreads = 256;

__global__ void __launch_bounds__(kEndpointThreads)
endpoint_update_kernel(const __grid_constant__ EndpointArgs a, const float *__restrict__ probs, long long pitch, int n, long long pos0) {
    const int r = blockIdx.x * kEndpointThreads + threadIdx.x;
    if (r < a.n_rows) endpoint_update_row(a, r, probs, pitch, n, pos0);
}

__global__ void __launch_bounds__(kEndpointThreads)
endpoint_arm_kernel(const __grid_constant__ EndpointArgs a, const __grid_constant__ EndpointReplay R, const int32_t *__restrict__ ids, int n) {
    const int i = blockIdx.x * kEndpointThreads + threadIdx.x;
    if (i < n) endpoint_arm_one(a, R, ids[i]);
}

// ids == nullptr: rows [0, n_rows); else the rows of the n listed global ids (ids outside the set ignored)
__global__ void __launch_bounds__(kEndpointThreads)
endpoint_clear_kernel(const __grid_constant__ EndpointArgs a, const int32_t *__restrict__ ids, int n, int reset) {
    const int i = blockIdx.x * kEndpointThreads + threadIdx.x;
    if (i >= n) return;
    const int r = ids ? endpoint_row(a, ids[i]) : i;
    if (r >= 0) endpoint_clear_row(a, r, reset);
}

// out [capacity][out_stride]: row i = the command of event slot i (endpoint_command_span), zeros past its length.  vec: units
// of 8 entries and 16-byte stores; a unit whose 8 samples lie in the ring, inside the length, from a slot that is a multiple of
// 8 (history_read_vec_shape) is one 16-byte load, any other unit is gathered a sample at a time.
__global__ void __launch_bounds__(kEndpointThreads)
endpoint_read_kernel(const int16_t *__restrict__ ring, int C, long long seen, const unsigned long long *__restrict__ count,
                     const mww_endpoint_event *__restrict__ events, int capacity, long long pre, long long post, int max_samples,
                     int16_t *__restrict__ out, long long out_stride, int32_t *__restrict__ lengths, int vec) {
    const long long used = (long long)*count;
    const int units = vec ? max_samples / 8 : max_samples;
    const int per_slot = units > 0 ? units : 1;          // max_samples 0 still writes every slot's length
    const long long total = (long long)capacity * per_slot;
    for (long long i = (long long)blockIdx.x * kEndpointThreads + threadIdx.x; i < total; i += (long long)gridDim.x * kEndpointThreads) {
        const int slot = (int)(i / per_slot);
        const int u = (int)(i - (long long)slot * per_slot);
        const CommandSpan c = endpoint_command_span(slot, used, capacity, events, pre, post, max_samples);
        if (u == 0) lengths[slot] = c.len;
        if (units == 0) continue;
        const int id = c.len > 0 ? events[slot].stream : 0;
        int16_t *dst = out + (long long)slot * out_stride;
        if (!vec) {
            dst[u] = u < c.len ? endpoint_command_one(ring, C, seen, id, c.a + u) : (int16_t)0;
            continue;
        }
        const int k0 = 8 * u;
        const long long t0 = c.a + k0;
        uint4 v = make_uint4(0, 0, 0, 0);
        if (k0 + 8 <= c.len && endpoint_in_ring(t0, seen, C) && endpoint_in_ring(t0 + 7, seen, C) &&
            history_read_vec_shape(history_mod(t0, C), max_samples, out_stride)) {
            v = *reinterpret_cast<const uint4 *>(ring + (long long)id * C + history_mod(t0, C));
        } else if (k0 < c.len) {
            uint32_t w[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int k = k0 + 2 * q;
                const int16_t lo = k < c.len ? endpoint_command_one(ring, C, seen, id, c.a + k) : (int16_t)0;
                const int16_t hi = k + 1 < c.len ? endpoint_command_one(ring, C, seen, id, c.a + k + 1) : (int16_t)0;
                w[q] = pack16(lo, hi);
            }
            v = make_uint4(w[0], w[1], w[2], w[3]);
        }
        *reinterpret_cast<uint4 *>(dst + k0) = v;
    }
}

unsigned endpoint_blocks(long long n) { return (unsigned)std::max<long long>(1, (n + kEndpointThreads - 1) / kEndpointThreads); }

}  // namespace

cudaError_t launch_endpoint_update(const EndpointArgs &a, const float *probs, long long pitch, int n, long long pos0, cudaStream_t st) {
    endpoint_update_kernel<<<endpoint_blocks(a.n_rows), kEndpointThreads, 0, st>>>(a, probs, pitch, n, pos0);
    return cudaGetLastError();
}

cudaError_t launch_endpoint_arm(const EndpointArgs &a, const EndpointReplay &R, const int32_t *ids, int n, cudaStream_t st) {
    endpoint_arm_kernel<<<endpoint_blocks(n), kEndpointThreads, 0, st>>>(a, R, ids, n);
    return cudaGetLastError();
}

cudaError_t launch_endpoint_clear(const EndpointArgs &a, const int32_t *ids, int n, int reset, cudaStream_t st) {
    endpoint_clear_kernel<<<endpoint_blocks(n), kEndpointThreads, 0, st>>>(a, ids, n, reset);
    return cudaGetLastError();
}

cudaError_t launch_endpoint_read(const int16_t *ring, int C, long long seen, const unsigned long long *count, const mww_endpoint_event *events,
                                 int capacity, long long pre, long long post, int max_samples, int16_t *out, long long out_stride,
                                 int32_t *lengths, int sm_count, cudaStream_t st) {
    const int vec = max_samples % 8 == 0 && out_stride % 8 == 0 && reinterpret_cast<uintptr_t>(out) % 16 == 0;
    const long long units = (long long)capacity * std::max(vec ? max_samples / 8 : max_samples, 1);
    const unsigned blocks = (unsigned)std::min<long long>(endpoint_blocks(units), (long long)sm_count * 16);
    endpoint_read_kernel<<<blocks, kEndpointThreads, 0, st>>>(ring, C, seen, count, events, capacity, pre, post, max_samples, out,
                                                              out_stride, lengths, vec);
    return cudaGetLastError();
}

}  // namespace mww
