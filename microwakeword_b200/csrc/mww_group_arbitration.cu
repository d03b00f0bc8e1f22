// mww_group_arbitration.cu -- the kernels of group arbitration (include/mww.h, "group arbitration"; spans, level, key and close
// in mww_group_arbitration.h): the arbitrated timed updates, which run the detectors' bodies (mww_detector.cuh,
// mww_detector_models.cuh) and offer a grouped row's events to its group with their level, and the close, which applies
// grouped detection's rule with the level order and appends the winners with their levels.  An update is these two launches
// whatever the number of events; a flush is the close alone.
//
// The level is measured where the offer happens, by the offering lane's whole warp: the sinks are called by whole warps
// (append_events, the models kernel's emit), so a ballot finds the offering lanes and the warp reads each one's Ls + Ln
// samples in turn, 8-sample units of 16 bytes per lane, and reduces the exact integer sums by shuffles.  A warp with no
// offering lane pays one ballot per step.  A companion library of its own, libmww_group_arbitration.so, so that every other
// library keeps exactly the kernels it had.
#include <math_constants.h>

#include "mww_detector.cuh"
#include "mww_detector_models.cuh"

namespace mww {

namespace {

constexpr int kArbitrationThreads = 256;

// sum x^2 and sum x of one 8-sample unit starting at position p (its 16 bytes `v`), over the positions in [lo, hi) and on
// either side of `split`: speech (>= split) and noise (< split)
MWW_D void unit_sums(uint4 v, long long p, const ArbitrationSpan &sp, unsigned long long &qs, long long &rs, unsigned long long &qn,
                     long long &rn) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const long long at = p + i;
        const int x = (at >= sp.lo && at < sp.hi) ? (int)(int16_t)(w[i >> 1] >> (16 * (i & 1))) : 0;
        const unsigned x2 = (unsigned)(x * x);
        if (at >= sp.split) { qs += x2; rs += x; }
        else { qn += x2; rn += x; }
    }
}

// the level of a candidate of `stream` at P, by the whole warp (every lane returns it)
MWW_D float warp_level(const ArbitrationArgs &r, int stream, long long P) {
    const ArbitrationSpan sp = arbitration_span(P, r.speech, r.noise, r.seen, r.capacity);
    const int lane = threadIdx.x & 31, C = r.capacity;
    unsigned long long qs = 0, qn = 0;
    long long rs = 0, rn = 0;
    if (sp.hi > sp.lo) {
        // units on positions that are multiples of 8 sit on slots that are multiples of 8 (C % 8 == 0): 16-byte loads that never
        // straddle the wrap.  C > 256, so one subtraction keeps the slot in the ring.
        const int16_t *row = r.ring + (long long)stream * C;
        long long p = (sp.lo & ~7LL) + 8 * lane;
        int slot = history_mod(p, C);
        for (; p < sp.hi; p += 256) {
            unit_sums(*reinterpret_cast<const uint4 *>(row + slot), p, sp, qs, rs, qn, rn);
            slot += 256;
            if (slot >= C) slot -= C;
        }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        qs += __shfl_xor_sync(kFull, qs, o); rs += __shfl_xor_sync(kFull, rs, o);
        qn += __shfl_xor_sync(kFull, qn, o); rn += __shfl_xor_sync(kFull, rn, o);
    }
    return arbitration_level(arbitration_energy(qs, rs, r.speech), arbitration_energy(qn, rn, r.noise));
}

// the levels of the warp's offering lanes, one after the other by the whole warp; 0 on the other lanes.  Called by whole warps.
MWW_D float warp_offer_levels(const ArbitrationArgs &r, bool offer, int stream, long long P) {
    unsigned todo = __ballot_sync(kFull, offer);
    const int lane = threadIdx.x & 31;
    float level = 0.f;
    while (todo) {
        const int src = __ffs(todo) - 1;
        todo &= todo - 1;
        const float l = warp_level(r, __shfl_sync(kFull, stream, src), __shfl_sync(kFull, P, src));
        if (lane == src) level = l;
    }
    return level;
}

// the plain detector's sink: a row of group -1 stores its event with its position and a NaN level; a row of a group offers it
// to the group's pending slot with its level
struct ArbitratedPositions {
    const GroupArgs &g;
    const ArbitrationArgs &r;
    long long last_end, step_samples;
    int n;
    static constexpr bool kOffers = true;
    MWW_D bool keep(const DetectorArgs &a, bool fire, int row, float score, int t) const {
        const int grp = fire ? g.groups[row] : -1;
        const bool offer = grp >= 0;
        const int32_t stream = offer ? (a.stream_ids ? a.stream_ids[row] : row) : 0;
        const float level = warp_offer_levels(r, offer, stream, event_step_end(last_end, step_samples, n, t));
        if (offer) group_offer(&g.pending[grp], arbitration_key(level, score, t, row), t);
        return fire && !offer;
    }
    MWW_D void put(unsigned long long slot, int t) const {
        g.positions[slot] = event_step_end(last_end, step_samples, n, t);
        g.ev_group[slot] = -1;
        g.ev_candidates[slot] = 1;
        r.ev_level[slot] = CUDART_NAN_F;
    }
};

template <bool kWarpPerRow, bool kRowCutoff>
__global__ void __launch_bounds__(kThreads)
detector_update_arbitrated_kernel(DetectorArgs a, const float *__restrict__ probs, int n_steps, long long pitch, const double *__restrict__ row_cutoff,
                                  const __grid_constant__ GroupArgs g, const __grid_constant__ ArbitrationArgs r, long long last_end,
                                  long long step_samples) {
    detector_update_rows<kWarpPerRow, kRowCutoff>(a, probs, n_steps, pitch, row_cutoff, ArbitratedPositions{g, r, last_end, step_samples, n_steps});
}

// the models kernel's sink, likewise per (group, WAKE model); the key's id is the global stream
template <typename M>
struct ArbitratedEmit {
    WarpEmit<M> emit;
    const GroupArgs &g;
    const ArbitrationArgs &r;
    long long row0_end;
    int hop;
    MWW_D void operator()(bool fire, int k, int stream, long long step, float score, int j) const {
        const DetectModelsArgsT<M> &a = emit.a;
        const int grp = fire ? g.groups[stream] : -1;
        const bool offer = grp >= 0;
        const long long P = event_model_step_end(row0_end, hop, j, a.models[k].stride, a.call[k].pending);
        const float level = warp_offer_levels(r, offer, stream, P);
        if (offer) group_offer(&g.pending[(long long)grp * g.n_wake + g.wake_of[k]], arbitration_key(level, score, j, stream), j);
        const long long slot = emit(fire && !offer, k, stream, step, score);
        if (slot < 0) return;
        g.positions[slot] = P;
        g.ev_group[slot] = -1;
        g.ev_candidates[slot] = 1;
        r.ev_level[slot] = CUDART_NAN_F;
    }
};

template <typename M>
__global__ void __launch_bounds__(kModelsThreads, 1)
detector_models_update_arbitrated_kernel(const __grid_constant__ DetectModelsArgsT<M> a, const __grid_constant__ GroupArgs g,
                                         const __grid_constant__ ArbitrationArgs r, long long row0_end, int hop) {
    const int stream = blockIdx.x * blockDim.x + threadIdx.x;          // lanes past n_streams stay for the ballots
    ArbitratedEmit<M> emit{WarpEmit<M>{a}, g, r, row0_end, hop};
    detect_models_stream(a, stream, emit);
}

// the warp's lanes whose `fire` is set append their group's winner with its level, as append_events appends: one atomicAdd for
// all of them, counted past capacity.  Called by whole warps.
MWW_D void append_arbitrated(unsigned long long *count, int capacity, mww_event *events, int32_t *fired, const GroupArgs &g,
                             const ArbitrationArgs &r, bool fire, const GroupEvent &e, int model, int grp) {
    const unsigned mask = __ballot_sync(kFull, fire);
    if (mask == 0) return;
    const int lane = threadIdx.x & 31;
    unsigned long long base = 0;
    if (lane == 0) base = atomicAdd(count, (unsigned long long)__popc(mask));
    base = __shfl_sync(kFull, base, 0);
    const unsigned long long slot = base + __popc(mask & ((1u << lane) - 1));
    if (!fire || slot >= (unsigned long long)capacity) return;
    mww_event ev;
    ev.stream = e.stream; ev.reserved = model; ev.step = e.step; ev.score = e.score; ev.pad = 0;
    events[slot] = ev;
    fired[slot] = e.stream;
    g.positions[slot] = e.sample;
    g.ev_group[slot] = grp;
    g.ev_candidates[slot] = e.candidates;
    r.ev_level[slot] = e.level;
}

__global__ void __launch_bounds__(kArbitrationThreads)
detector_arbitrated_close_kernel(DetectorArgs a, const __grid_constant__ GroupArgs g, const __grid_constant__ ArbitrationArgs r, long long last_end,
                                 long long step_samples, int n, int flush) {
    const int s = blockIdx.x * kArbitrationThreads + threadIdx.x;       // idle lanes stay for the ballots
    GroupClosed c;
    if (s < g.n_slots) {
        auto pos = [&](int t) { return event_step_end(last_end, step_samples, n, t); };
        auto seen = [&](int row) { return a.seen[row]; };
        auto stream = [&](int row) { return a.stream_ids ? a.stream_ids[row] : row; };
        c = arbitration_close_slot(g.pending, g.windows, r.levels, g.window, s, n, pos, seen, stream, last_end + step_samples, flush != 0);
    }
    append_arbitrated(a.count, a.capacity, a.events, a.fired, g, r, c.first, c.e1, 0, s);
    append_arbitrated(a.count, a.capacity, a.events, a.fired, g, r, c.second, c.e2, 0, s);
}

__global__ void __launch_bounds__(kArbitrationThreads)
detector_models_arbitrated_close_kernel(const __grid_constant__ DetectModelsArgs a, const __grid_constant__ GroupArgs g,
                                        const __grid_constant__ ArbitrationArgs r, long long row0_end, long long row_end, int hop, int flush) {
    const int s = blockIdx.x * kArbitrationThreads + threadIdx.x;
    GroupClosed c;
    int k = 0, grp = 0;
    if (s < g.n_slots) {
        grp = s / g.n_wake;
        k = a.wake[s - grp * g.n_wake];
        const DetectModel &m = a.models[k];
        const DetectCall &call = a.call[k];
        auto pos = [&](int j) { return event_model_step_end(row0_end, hop, j, m.stride, call.pending); };
        auto seen = [&](int stream) { return m.seen[detect_row(m, stream, a.n_streams)]; };
        auto same = [](int stream) { return stream; };
        c = arbitration_close_slot(g.pending, g.windows, r.levels, g.window, s, flush ? 0 : call.n_steps, pos, seen, same, row_end + hop, flush != 0);
    }
    append_arbitrated(a.count, a.capacity, a.events, a.fired, g, r, c.first, c.e1, k, grp);
    append_arbitrated(a.count, a.capacity, a.events, a.fired, g, r, c.second, c.e2, k, grp);
}

unsigned arbitration_blocks(int n_slots) { return (unsigned)((n_slots + kArbitrationThreads - 1) / kArbitrationThreads); }

template <typename M>
cudaError_t launch_models_arbitrated(const DetectModelsArgsT<M> &a, const DetectModelsArgs &base, const GroupArgs &g, const ArbitrationArgs &r,
                                     long long row0_end, long long row_end, int hop, cudaStream_t st) {
    if (a.n_streams <= 0) return cudaSuccess;
    detector_models_update_arbitrated_kernel<M><<<(unsigned)((a.n_streams + kModelsThreads - 1) / kModelsThreads), kModelsThreads, 0, st>>>(
        a, g, r, row0_end, hop);
    detector_models_arbitrated_close_kernel<<<arbitration_blocks(g.n_slots), kArbitrationThreads, 0, st>>>(base, g, r, row0_end, row_end, hop, 0);
    return cudaGetLastError();
}

}  // namespace

cudaError_t launch_detector_update_arbitrated(const DetectorArgs &a, const double *row_cutoff, const float *probs, int n_steps, long long pitch,
                                              const GroupArgs &g, const ArbitrationArgs &r, long long last_end, long long step_samples,
                                              cudaStream_t st) {
    if (n_steps <= 0 || a.n_rows <= 0) return cudaSuccess;
    const unsigned blocks = update_form_blocks(a, n_steps);
    const bool warp = n_steps >= kDetectorWarpMinSteps;
    if (row_cutoff) {
        if (warp) detector_update_arbitrated_kernel<true, true><<<blocks, kThreads, 0, st>>>(a, probs, n_steps, pitch, row_cutoff, g, r, last_end, step_samples);
        else detector_update_arbitrated_kernel<false, true><<<blocks, kThreads, 0, st>>>(a, probs, n_steps, pitch, row_cutoff, g, r, last_end, step_samples);
    } else {
        if (warp) detector_update_arbitrated_kernel<true, false><<<blocks, kThreads, 0, st>>>(a, probs, n_steps, pitch, nullptr, g, r, last_end, step_samples);
        else detector_update_arbitrated_kernel<false, false><<<blocks, kThreads, 0, st>>>(a, probs, n_steps, pitch, nullptr, g, r, last_end, step_samples);
    }
    detector_arbitrated_close_kernel<<<arbitration_blocks(g.n_slots), kArbitrationThreads, 0, st>>>(a, g, r, last_end, step_samples, n_steps, 0);
    return cudaGetLastError();
}

cudaError_t launch_detector_models_update_arbitrated(const DetectModelsArgs &a, const GroupArgs &g, const ArbitrationArgs &r, long long row0_end,
                                                     long long row_end, int hop, cudaStream_t st) {
    return launch_models_arbitrated(a, a, g, r, row0_end, row_end, hop, st);
}
cudaError_t launch_detector_models_update_arbitrated(const DetectModelsArgsT<DetectModelRows> &a, const DetectModelsArgs &base, const GroupArgs &g,
                                                     const ArbitrationArgs &r, long long row0_end, long long row_end, int hop, cudaStream_t st) {
    return launch_models_arbitrated(a, base, g, r, row0_end, row_end, hop, st);
}

cudaError_t launch_detector_arbitrated_flush(const DetectorArgs &a, const GroupArgs &g, const ArbitrationArgs &r, cudaStream_t st) {
    detector_arbitrated_close_kernel<<<arbitration_blocks(g.n_slots), kArbitrationThreads, 0, st>>>(a, g, r, 0, 1, 0, 1);
    return cudaGetLastError();
}
cudaError_t launch_detector_models_arbitrated_flush(const DetectModelsArgs &a, const GroupArgs &g, const ArbitrationArgs &r, cudaStream_t st) {
    detector_models_arbitrated_close_kernel<<<arbitration_blocks(g.n_slots), kArbitrationThreads, 0, st>>>(a, g, r, 0, 0, 0, 1);
    return cudaGetLastError();
}

}  // namespace mww
