// mww_detector_models.cuh -- the multi-model streaming detector's update kernel (rule and per-stream body:
// mww_detector_models.h), included by mww_detector_models.cu (uniform mode), mww_detector_cutoffs.cu (per-row mode,
// mww_set_multi_detector_cutoffs) and mww_event_positions.cu (the timed kernel, whose emit also stores each event's position).
//
// detector_models_update_kernel: a thread per global stream walks the call's steps of the VAD and of every WAKE model it
// belongs to (detect_models_stream).  Each model's state is struct-of-arrays over its members, so for a model on all
// streams the row is the stream and every access of a warp is one coalesced line; a model with a stream set reads its
// rows through the inverse map.  The loops' bounds depend on the call only, never on the stream, so every lane of a warp
// reaches every WAKE step together and events go to the shared buffer through one atomicAdd per warp.  With per-row
// descriptors (DetectModelRows) the VAD row's cutoff is loaded once per call, and a WAKE row's with its seen and cooldown:
// once per VAD step that has WAKE steps ending before it (once per call without a VAD or in a live call).
#pragma once

#include <cuda_runtime.h>

#include "mww_kernels.h"

namespace mww {

namespace {

constexpr unsigned kModelsFull = 0xffffffffu;
constexpr int kModelsThreads = 256;

// the warp's lanes whose `fire` is set append one event each: one atomicAdd for all of them.  Called by whole warps.
// -> the slot of a stored event, -1 otherwise.
template <typename M>
struct WarpEmit {
    const DetectModelsArgsT<M> &a;
    MWW_D long long operator()(bool fire, int k, int stream, long long step, float score) const {
        const unsigned mask = __ballot_sync(kModelsFull, fire);
        if (mask == 0) return -1;
        const int lane = threadIdx.x & 31;
        unsigned long long base = 0;
        if (lane == 0) base = atomicAdd(a.count, (unsigned long long)__popc(mask));
        base = __shfl_sync(kModelsFull, base, 0);
        const unsigned long long slot = base + __popc(mask & ((1u << lane) - 1));
        if (!fire || slot >= (unsigned long long)a.capacity) return -1;   // past capacity: counted, not stored
        mww_event e;
        e.stream = stream; e.reserved = k; e.step = step; e.score = score; e.pad = 0;
        a.events[slot] = e;
        a.fired[slot] = stream;
        return (long long)slot;
    }
};

}  // namespace

// M: DetectModel (the rule's cutoff) or DetectModelRows (each row's)
template <typename M>
__global__ void __launch_bounds__(kModelsThreads) detector_models_update_kernel(const __grid_constant__ DetectModelsArgsT<M> a) {
    const int stream = blockIdx.x * blockDim.x + threadIdx.x;          // lanes past n_streams stay for the ballots
    WarpEmit<M> emit{a};
    detect_models_stream(a, stream, emit);
}

template <typename M>
cudaError_t launch_models_update_form(const DetectModelsArgsT<M> &a, cudaStream_t st) {
    if (a.n_streams <= 0) return cudaSuccess;
    detector_models_update_kernel<M><<<(unsigned)((a.n_streams + kModelsThreads - 1) / kModelsThreads), kModelsThreads, 0, st>>>(a);
    return cudaGetLastError();
}

}  // namespace mww
