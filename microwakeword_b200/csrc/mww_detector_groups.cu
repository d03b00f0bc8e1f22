// mww_detector_groups.cu -- the kernels of grouped detection (include/mww.h, "grouped detection"; key, offer and close in
// mww_detector_groups.h): the grouped timed updates, which run the detectors' bodies (mww_detector.cuh,
// mww_detector_models.cuh) and offer a grouped row's events to its group instead of storing them, and the close, which applies
// the rule to every group slot after the update and appends the winners.  An update is these two launches whatever the number
// of events; a flush is the close alone.  A thread per group slot: the close reads 32 + 40 bytes per slot, which at 16 384
// groups is less than the update's own traffic at 65 536 rows (DESIGN.md section 4).  A companion library of its own,
// libmww_detector_groups.so, so that every other library keeps exactly the kernels it had.
#include <climits>

#include "mww_detector.cuh"
#include "mww_detector_models.cuh"

namespace mww {

namespace {

constexpr int kGroupThreads = 256;

// the plain detector's sink: a row of group -1 stores its event with its position, as the timed detector does; a row of a
// group offers it to the group's pending slot
struct GroupedPositions {
    const GroupArgs &g;
    long long last_end, step_samples;
    int n;
    static constexpr bool kOffers = true;
    MWW_D bool keep(const DetectorArgs &a, bool fire, int row, float score, int t) const {
        if (!fire) return false;
        const int grp = g.groups[row];
        if (grp < 0) return true;
        group_offer(&g.pending[grp], group_key(score, t, a.stream_ids ? a.stream_ids[row] : row, row), t);
        return false;
    }
    MWW_D void put(unsigned long long slot, int t) const {
        g.positions[slot] = event_step_end(last_end, step_samples, n, t);
        g.ev_group[slot] = -1;
        g.ev_candidates[slot] = 1;
    }
};

template <bool kWarpPerRow, bool kRowCutoff>
__global__ void __launch_bounds__(kThreads)
detector_update_grouped_kernel(DetectorArgs a, const float *__restrict__ probs, int n_steps, long long pitch, const double *__restrict__ row_cutoff,
                               const __grid_constant__ GroupArgs g, long long last_end, long long step_samples) {
    detector_update_rows<kWarpPerRow, kRowCutoff>(a, probs, n_steps, pitch, row_cutoff, GroupedPositions{g, last_end, step_samples, n_steps});
}

// the models kernel's sink, likewise per (group, WAKE model)
template <typename M>
struct GroupedEmit {
    WarpEmit<M> emit;
    const GroupArgs &g;
    long long row0_end;
    int hop;
    MWW_D void operator()(bool fire, int k, int stream, long long step, float score, int j) const {
        const DetectModelsArgsT<M> &a = emit.a;
        bool store = fire;
        if (fire) {
            const int grp = g.groups[stream];
            if (grp >= 0) {
                store = false;
                group_offer(&g.pending[(long long)grp * g.n_wake + g.wake_of[k]], group_key(score, j, stream, detect_row(a.models[k], stream, a.n_streams)), j);
            }
        }
        const long long slot = emit(store, k, stream, step, score);
        if (slot < 0) return;
        g.positions[slot] = event_model_step_end(row0_end, hop, j, a.models[k].stride, a.call[k].pending);
        g.ev_group[slot] = -1;
        g.ev_candidates[slot] = 1;
    }
};

// one block per SM at least, so that ptxas takes the registers it needs (72) rather than spill around the offer
template <typename M>
__global__ void __launch_bounds__(kModelsThreads, 1)
detector_models_update_grouped_kernel(const __grid_constant__ DetectModelsArgsT<M> a, const __grid_constant__ GroupArgs g, long long row0_end, int hop) {
    const int stream = blockIdx.x * blockDim.x + threadIdx.x;          // lanes past n_streams stay for the ballots
    GroupedEmit<M> emit{WarpEmit<M>{a}, g, row0_end, hop};
    detect_models_stream(a, stream, emit);
}

// the warp's lanes whose `fire` is set append their group's winner, as append_events appends: one atomicAdd for all of them,
// counted past capacity.  Called by whole warps.
MWW_D void append_winners(unsigned long long *count, int capacity, mww_event *events, int32_t *fired, const GroupArgs &g, bool fire,
                          const GroupEvent &e, int model, int grp) {
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
}

// one slot's close: its pending offers resolved with the call's clock (position of step t: pos(t); step of row r: the row's seen
// after the call, minus the call's n steps, plus t), the rule applied, the pending slot cleared
template <typename Pos, typename Seen>
MWW_D GroupClosed close_slot(const GroupArgs &g, int s, int n, const Pos &pos, const Seen &seen, long long E, bool flush) {
    const GroupPending p = g.pending[s];
    GroupEvent best;
    long long p_min = 0;
    if (p.count) {
        const int t = group_key_t(p.best);
        best.stream = group_key_stream(p.best);
        best.score = group_key_score(p.best);
        best.sample = pos(t);
        best.step = seen(group_key_row(p.best)) - n + t;
        p_min = pos((int)p.tmin);
        g.pending[s] = GroupPending{};
    }
    mww_group_window w = g.windows[s];
    const GroupClosed c = group_close(w, p.count, best, p_min, !flush && n > 0, n > 0 ? pos(0) : 0, flush ? LLONG_MAX : E, g.window);
    if (p.count || c.first || c.second) g.windows[s] = w;
    return c;
}

__global__ void __launch_bounds__(kGroupThreads)
detector_groups_close_kernel(DetectorArgs a, const __grid_constant__ GroupArgs g, long long last_end, long long step_samples, int n, int flush) {
    const int s = blockIdx.x * kGroupThreads + threadIdx.x;             // idle lanes stay for the ballots
    GroupClosed c;
    if (s < g.n_slots) {
        auto pos = [&](int t) { return event_step_end(last_end, step_samples, n, t); };
        auto seen = [&](int row) { return a.seen[row]; };
        c = close_slot(g, s, n, pos, seen, last_end + step_samples, flush != 0);
    }
    append_winners(a.count, a.capacity, a.events, a.fired, g, c.first, c.e1, 0, s);
    append_winners(a.count, a.capacity, a.events, a.fired, g, c.second, c.e2, 0, s);
}

__global__ void __launch_bounds__(kGroupThreads)
detector_models_groups_close_kernel(const __grid_constant__ DetectModelsArgs a, const __grid_constant__ GroupArgs g, long long row0_end,
                                    long long row_end, int hop, int flush) {
    const int s = blockIdx.x * kGroupThreads + threadIdx.x;
    GroupClosed c;
    int k = 0, grp = 0;
    if (s < g.n_slots) {
        grp = s / g.n_wake;
        k = a.wake[s - grp * g.n_wake];
        const DetectModel &m = a.models[k];
        const DetectCall &call = a.call[k];
        auto pos = [&](int j) { return event_model_step_end(row0_end, hop, j, m.stride, call.pending); };
        auto seen = [&](int row) { return m.seen[row]; };
        c = close_slot(g, s, flush ? 0 : call.n_steps, pos, seen, row_end + hop, flush != 0);
    }
    append_winners(a.count, a.capacity, a.events, a.fired, g, c.first, c.e1, k, grp);
    append_winners(a.count, a.capacity, a.events, a.fired, g, c.second, c.e2, k, grp);
}

unsigned group_blocks(int n_slots) { return (unsigned)((n_slots + kGroupThreads - 1) / kGroupThreads); }

template <typename M>
cudaError_t launch_models_grouped(const DetectModelsArgsT<M> &a, const DetectModelsArgs &base, const GroupArgs &g, long long row0_end,
                                  long long row_end, int hop, cudaStream_t st) {
    if (a.n_streams <= 0) return cudaSuccess;
    detector_models_update_grouped_kernel<M><<<(unsigned)((a.n_streams + kModelsThreads - 1) / kModelsThreads), kModelsThreads, 0, st>>>(a, g, row0_end,
                                                                                                                                      hop);
    detector_models_groups_close_kernel<<<group_blocks(g.n_slots), kGroupThreads, 0, st>>>(base, g, row0_end, row_end, hop, 0);
    return cudaGetLastError();
}

}  // namespace

cudaError_t launch_detector_update_grouped(const DetectorArgs &a, const double *row_cutoff, const float *probs, int n_steps, long long pitch,
                                           const GroupArgs &g, long long last_end, long long step_samples, cudaStream_t st) {
    if (n_steps <= 0 || a.n_rows <= 0) return cudaSuccess;
    const unsigned blocks = update_form_blocks(a, n_steps);
    const bool warp = n_steps >= kDetectorWarpMinSteps;
    if (row_cutoff) {
        if (warp) detector_update_grouped_kernel<true, true><<<blocks, kThreads, 0, st>>>(a, probs, n_steps, pitch, row_cutoff, g, last_end, step_samples);
        else detector_update_grouped_kernel<false, true><<<blocks, kThreads, 0, st>>>(a, probs, n_steps, pitch, row_cutoff, g, last_end, step_samples);
    } else {
        if (warp) detector_update_grouped_kernel<true, false><<<blocks, kThreads, 0, st>>>(a, probs, n_steps, pitch, nullptr, g, last_end, step_samples);
        else detector_update_grouped_kernel<false, false><<<blocks, kThreads, 0, st>>>(a, probs, n_steps, pitch, nullptr, g, last_end, step_samples);
    }
    detector_groups_close_kernel<<<group_blocks(g.n_slots), kGroupThreads, 0, st>>>(a, g, last_end, step_samples, n_steps, 0);
    return cudaGetLastError();
}

cudaError_t launch_detector_models_update_grouped(const DetectModelsArgs &a, const GroupArgs &g, long long row0_end, long long row_end, int hop,
                                                  cudaStream_t st) {
    return launch_models_grouped(a, a, g, row0_end, row_end, hop, st);
}
cudaError_t launch_detector_models_update_grouped(const DetectModelsArgsT<DetectModelRows> &a, const DetectModelsArgs &base, const GroupArgs &g,
                                                  long long row0_end, long long row_end, int hop, cudaStream_t st) {
    return launch_models_grouped(a, base, g, row0_end, row_end, hop, st);
}

cudaError_t launch_detector_groups_flush(const DetectorArgs &a, const GroupArgs &g, cudaStream_t st) {
    detector_groups_close_kernel<<<group_blocks(g.n_slots), kGroupThreads, 0, st>>>(a, g, 0, 1, 0, 1);
    return cudaGetLastError();
}
cudaError_t launch_detector_models_groups_flush(const DetectModelsArgs &a, const GroupArgs &g, cudaStream_t st) {
    detector_models_groups_close_kernel<<<group_blocks(g.n_slots), kGroupThreads, 0, st>>>(a, g, 0, 0, 0, 1);
    return cudaGetLastError();
}

}  // namespace mww
