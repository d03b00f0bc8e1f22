// mww_detector_models.cu -- the multi-model streaming detector's kernels (rule and per-stream body: mww_detector_models.h).
//
// detector_models_update_kernel: a thread per global stream walks the call's steps of the VAD and of every WAKE model it
// belongs to (detect_models_stream).  Each model's state is struct-of-arrays over its members, so for a model on all
// streams the row is the stream and every access of a warp is one coalesced line; a model with a stream set reads its
// rows through the inverse map.  The loops' bounds depend on the call only, never on the stream, so every lane of a warp
// reaches every WAKE step together and events go to the shared buffer through one atomicAdd per warp.
// detector_models_reset_kernel: a thread per listed stream resets that stream's row of every model.
#include <cuda_runtime.h>

#include "mww_kernels.h"

namespace mww {

namespace {

constexpr unsigned kFull = 0xffffffffu;
constexpr int kThreads = 256;

// the warp's lanes whose `fire` is set append one event each: one atomicAdd for all of them.  Called by whole warps.
struct WarpEmit {
    const DetectModelsArgs &a;
    MWW_D void operator()(bool fire, int k, int stream, long long step, float score) const {
        const unsigned mask = __ballot_sync(kFull, fire);
        if (mask == 0) return;
        const int lane = threadIdx.x & 31;
        unsigned long long base = 0;
        if (lane == 0) base = atomicAdd(a.count, (unsigned long long)__popc(mask));
        base = __shfl_sync(kFull, base, 0);
        const unsigned long long slot = base + __popc(mask & ((1u << lane) - 1));
        if (!fire || slot >= (unsigned long long)a.capacity) return;      // past capacity: counted, not stored
        mww_event e;
        e.stream = stream; e.reserved = k; e.step = step; e.score = score; e.pad = 0;
        a.events[slot] = e;
        a.fired[slot] = stream;
    }
};

}  // namespace

__global__ void __launch_bounds__(kThreads) detector_models_update_kernel(const __grid_constant__ DetectModelsArgs a) {
    const int stream = blockIdx.x * blockDim.x + threadIdx.x;          // lanes past n_streams stay for the ballots
    WarpEmit emit{a};
    detect_models_stream(a, stream, emit);
}

// fresh state for the streams ids[0, n) (out of range ignored) or, ids == nullptr, for streams [0, n)
__global__ void __launch_bounds__(kThreads) detector_models_reset_kernel(const __grid_constant__ DetectModelsArgs a,
                                                                         const int32_t *__restrict__ ids, int n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    detect_models_reset_stream(a, ids ? ids[i] : i);
}

cudaError_t launch_detector_models_update(const DetectModelsArgs &a, cudaStream_t st) {
    if (a.n_streams <= 0) return cudaSuccess;
    detector_models_update_kernel<<<(unsigned)((a.n_streams + kThreads - 1) / kThreads), kThreads, 0, st>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_detector_models_reset(const DetectModelsArgs &a, const int32_t *ids, int n, cudaStream_t st) {
    if (n <= 0) return cudaSuccess;
    detector_models_reset_kernel<<<(unsigned)((n + kThreads - 1) / kThreads), kThreads, 0, st>>>(a, ids, n);
    return cudaGetLastError();
}

}  // namespace mww
