// mww_event_positions.cu -- the kernels of event positions (include/mww.h, "event positions"; positions and bodies in
// mww_event_positions.h): the timed detectors' updates, which run the untimed kernels' bodies (mww_detector.cuh,
// mww_detector_models.cuh) and store one int64 beside each event they store; the history read that ends at given positions;
// and the verifier slots that end at their events.  A companion library of its own, libmww_event_positions.so, so that
// libmww_b200.so and the other companion libraries keep exactly the kernels they had.
#include <algorithm>

#include "mww_detector.cuh"
#include "mww_detector_models.cuh"

namespace mww {

namespace {

constexpr int kPositionsThreads = 256;

// the plain detector's clock: an event of step t of the call is placed at event_step_end
struct StepPositions {
    long long *out;
    long long last_end, step_samples;
    int n;
    static constexpr bool kOffers = false;
    MWW_D void put(unsigned long long slot, int t) const { out[slot] = event_step_end(last_end, step_samples, n, t); }
};

template <bool kWarpPerRow, bool kRowCutoff>
__global__ void __launch_bounds__(kThreads)
detector_update_at_kernel(DetectorArgs a, const float *__restrict__ probs, int n_steps, long long pitch, const double *__restrict__ row_cutoff,
                          long long *__restrict__ positions, long long last_end, long long step_samples) {
    detector_update_rows<kWarpPerRow, kRowCutoff>(a, probs, n_steps, pitch, row_cutoff, StepPositions{positions, last_end, step_samples, n_steps});
}

// the models kernel's emit, and the position of each event it stores: WAKE step j of model k at event_model_step_end
template <typename M>
struct TimedEmit {
    WarpEmit<M> emit;
    long long *out;
    long long row0_end;
    int hop;
    MWW_D void operator()(bool fire, int k, int stream, long long step, float score, int j) const {
        const long long slot = emit(fire, k, stream, step, score);
        if (slot >= 0) out[slot] = event_model_step_end(row0_end, hop, j, emit.a.models[k].stride, emit.a.call[k].pending);
    }
};

template <typename M>
__global__ void __launch_bounds__(kModelsThreads)
detector_models_update_at_kernel(const __grid_constant__ DetectModelsArgsT<M> a, long long *__restrict__ positions, long long row0_end, int hop) {
    const int stream = blockIdx.x * blockDim.x + threadIdx.x;          // lanes past n_streams stay for the ballots
    TimedEmit<M> emit{WarpEmit<M>{a}, positions, row0_end, hop};
    detect_models_stream(a, stream, emit);
}

// n rows of n_samples: row i ends at ends[i] (history_at_one).  vec: units of 8 entries and 16-byte stores; a unit whose 8
// samples are in the ring from a slot that is a multiple of 8 is one 16-byte load, any other unit is gathered a sample at a time
// -- the endpointer's command read, with a row's start at ends[i] - n_samples.
__global__ void __launch_bounds__(kPositionsThreads)
history_read_at_kernel(const int16_t *__restrict__ ring, int C, long long seen, const int32_t *__restrict__ ids, const long long *__restrict__ ends,
                       int n, int n_streams, int n_samples, int16_t *__restrict__ out, long long out_stride, int vec) {
    const int units = vec ? n_samples / 8 : n_samples;
    const long long total = (long long)n * units;
    for (long long i = (long long)blockIdx.x * kPositionsThreads + threadIdx.x; i < total; i += (long long)gridDim.x * kPositionsThreads) {
        const long long r = i / units;
        const int u = (int)(i - r * units);
        const int id = ids[r];
        const long long end = ends[r];
        int16_t *dst = out + r * out_stride;
        if (!vec) {
            dst[u] = history_at_one(ring, C, seen, id, n_streams, end, n_samples, u);
            continue;
        }
        const int k0 = 8 * u;
        uint4 v;
        if (history_at_unit_in_ring(seen, C, id, n_streams, end, n_samples, u, out_stride)) {
            v = *reinterpret_cast<const uint4 *>(ring + (long long)id * C + history_mod(end - n_samples + k0, C));
        } else {
            uint32_t w[4];
#pragma unroll
            for (int q = 0; q < 4; ++q)
                w[q] = pack16(history_at_one(ring, C, seen, id, n_streams, end, n_samples, k0 + 2 * q),
                              history_at_one(ring, C, seen, id, n_streams, end, n_samples, k0 + 2 * q + 1));
            v = make_uint4(w[0], w[1], w[2], w[3]);
        }
        *reinterpret_cast<uint4 *>(dst + k0) = v;
    }
}

__global__ void __launch_bounds__(kPositionsThreads)
verify_slots_at_kernel(const long long *__restrict__ count, const mww_event *__restrict__ events, const long long *__restrict__ positions,
                       int capacity, int model, long long post, long long seen, int C, int n_samples, int32_t *__restrict__ ids,
                       long long *__restrict__ ends) {
    const int i = blockIdx.x * kPositionsThreads + threadIdx.x;
    if (i >= capacity) return;
    const SlotAt s = verify_slot_at(i, *count, capacity, events, positions, model, post, seen, C, n_samples);
    ids[i] = s.id;
    ends[i] = s.end;
}

unsigned positions_blocks(long long n) { return (unsigned)std::max<long long>(1, (n + kPositionsThreads - 1) / kPositionsThreads); }

template <typename M>
cudaError_t launch_models_at(const DetectModelsArgsT<M> &a, long long *positions, long long row0_end, int hop, cudaStream_t st) {
    if (a.n_streams <= 0) return cudaSuccess;
    detector_models_update_at_kernel<M><<<(unsigned)((a.n_streams + kModelsThreads - 1) / kModelsThreads), kModelsThreads, 0, st>>>(a, positions,
                                                                                                                                 row0_end, hop);
    return cudaGetLastError();
}

}  // namespace

cudaError_t launch_detector_update_at(const DetectorArgs &a, const double *row_cutoff, const float *probs, int n_steps, long long pitch,
                                      long long *positions, long long last_end, long long step_samples, cudaStream_t st) {
    if (n_steps <= 0 || a.n_rows <= 0) return cudaSuccess;
    const unsigned blocks = update_form_blocks(a, n_steps);
    const bool warp = n_steps >= kDetectorWarpMinSteps;
    if (row_cutoff) {
        if (warp) detector_update_at_kernel<true, true><<<blocks, kThreads, 0, st>>>(a, probs, n_steps, pitch, row_cutoff, positions, last_end, step_samples);
        else detector_update_at_kernel<false, true><<<blocks, kThreads, 0, st>>>(a, probs, n_steps, pitch, row_cutoff, positions, last_end, step_samples);
    } else {
        if (warp) detector_update_at_kernel<true, false><<<blocks, kThreads, 0, st>>>(a, probs, n_steps, pitch, nullptr, positions, last_end, step_samples);
        else detector_update_at_kernel<false, false><<<blocks, kThreads, 0, st>>>(a, probs, n_steps, pitch, nullptr, positions, last_end, step_samples);
    }
    return cudaGetLastError();
}

cudaError_t launch_detector_models_update_at(const DetectModelsArgs &a, long long *positions, long long row0_end, int hop, cudaStream_t st) {
    return launch_models_at(a, positions, row0_end, hop, st);
}
cudaError_t launch_detector_models_update_at(const DetectModelsArgsT<DetectModelRows> &a, long long *positions, long long row0_end, int hop,
                                             cudaStream_t st) {
    return launch_models_at(a, positions, row0_end, hop, st);
}

cudaError_t launch_history_read_at(const int16_t *ring, int C, long long seen, const int32_t *ids, const long long *ends, int n, int n_streams,
                                   int n_samples, int16_t *out, long long out_stride, int sm_count, cudaStream_t st) {
    if (n <= 0 || n_samples <= 0) return cudaSuccess;
    const int vec = n_samples % 8 == 0 && out_stride % 8 == 0 && reinterpret_cast<uintptr_t>(out) % 16 == 0;
    const long long total = (long long)n * (vec ? n_samples / 8 : n_samples);
    const unsigned blocks = (unsigned)std::min<long long>(positions_blocks(total), (long long)sm_count * 16);
    history_read_at_kernel<<<blocks, kPositionsThreads, 0, st>>>(ring, C, seen, ids, ends, n, n_streams, n_samples, out, out_stride, vec);
    return cudaGetLastError();
}

cudaError_t launch_verify_slots_at(const long long *count, const mww_event *events, const long long *positions, int capacity, int model,
                                   long long post, long long seen, int C, int n_samples, int32_t *ids, long long *ends, cudaStream_t st) {
    if (capacity <= 0) return cudaSuccess;
    verify_slots_at_kernel<<<positions_blocks(capacity), kPositionsThreads, 0, st>>>(count, events, positions, capacity, model, post, seen, C,
                                                                                     n_samples, ids, ends);
    return cudaGetLastError();
}

}  // namespace mww
