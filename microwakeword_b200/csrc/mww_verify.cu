// mww_verify.cu -- the two kernels of second-stage verification (per-element bodies: mww_verify.h): a detector's event
// slots to stream ids, read on the device so that the host never waits for the event count, and the verifier's scores to
// confirmed stream ids.  A thread per slot or index, so each is one launch whatever the count.  A companion library of its
// own, libmww_verify.so, so that libmww_b200.so and the other companion libraries keep exactly the kernels they had.
#include "mww_kernels.h"

namespace mww {

namespace {

constexpr int kVerifyThreads = 256;

__global__ void __launch_bounds__(kVerifyThreads)
verify_slots_kernel(const long long *__restrict__ count, const mww_event *__restrict__ events, int capacity, int model,
                    int32_t *__restrict__ ids) {
    const int i = blockIdx.x * kVerifyThreads + threadIdx.x;
    if (i < capacity) ids[i] = verify_slot_id(i, *count, capacity, events, model);
}

__global__ void __launch_bounds__(kVerifyThreads)
verify_confirm_kernel(const int32_t *__restrict__ ids, int n, int n_streams, const float *__restrict__ scores, double cutoff,
                      float *__restrict__ out_scores, int32_t *__restrict__ out_confirmed) {
    const int i = blockIdx.x * kVerifyThreads + threadIdx.x;
    if (i >= n) return;
    const VerifyOut o = verify_confirm(ids[i], n_streams, scores[i], cutoff);
    if (out_scores) out_scores[i] = o.score;
    if (out_confirmed) out_confirmed[i] = o.confirmed;
}

unsigned verify_blocks(int n) { return (unsigned)((n + kVerifyThreads - 1) / kVerifyThreads); }

}  // namespace

cudaError_t launch_verify_slots(const long long *count, const mww_event *events, int capacity, int model, int32_t *ids, cudaStream_t st) {
    if (capacity <= 0) return cudaSuccess;
    verify_slots_kernel<<<verify_blocks(capacity), kVerifyThreads, 0, st>>>(count, events, capacity, model, ids);
    return cudaGetLastError();
}

cudaError_t launch_verify_confirm(const int32_t *ids, int n, int n_streams, const float *scores, double cutoff, float *out_scores,
                                  int32_t *out_confirmed, cudaStream_t st) {
    if (n <= 0) return cudaSuccess;
    verify_confirm_kernel<<<verify_blocks(n), kVerifyThreads, 0, st>>>(ids, n, n_streams, scores, cutoff, out_scores, out_confirmed);
    return cudaGetLastError();
}

}  // namespace mww
