// mww_detector.cuh -- the streaming detector's update kernel (rule and both forms: mww_detector.h), included by
// mww_detector.cu (uniform cutoff), mww_detector_cutoffs.cu (per-row cutoffs, mww_set_detector_cutoffs) and
// mww_event_positions.cu (the timed kernels, which run the same body and also store each event's position) and
// mww_detector_groups.cu (the grouped kernels, which offer a grouped row's events to its group).
//
// detector_update_kernel<false, *>, thread per row: the live shape, one or a few steps for very many rows.  State is
// struct-of-arrays and the history [window - 1][n_rows], so every access of a warp is one coalesced line; a one-step call
// moves 8 (window - 1) + 28 bytes per row (history, counter and cooldown read and written, one probability read), and
// 8 more in per-row mode (the row's cutoff, read once per call, coalesced).
// detector_update_kernel<true, *>, warp per row: the clip shape, many steps per row.  32 consecutive steps per pass are loaded
// coalesced; the window - 1 values before them come from the history on the first pass and from the previous pass's
// registers afterwards, by shuffles; every lane forms one average and detector_chain_pass walks the cooldown chain.  In
// per-row mode every lane reads the row's cutoff once per call (one broadcast load per warp) and the ballot compares
// against it.
// Events go to the shared buffer through one atomicAdd per warp.
#pragma once

#include <cuda_runtime.h>

#include "mww_kernels.h"

namespace mww {

namespace {

constexpr unsigned kFull = 0xffffffffu;
constexpr int kThreads = 256;

// history of one row in global memory, entry j at hist[j * n_rows]
struct RowHistory {
    float *h; long long stride;
    MWW_D float get(int j) const { return h[j * stride]; }
    MWW_D void set(int j, float v) { h[j * stride] = v; }
};

// steps of a pass and the one before it, spread over the lanes: x(i) is step i of the pass for i >= 0 and step 32 + i of
// the previous pass for i < 0.  Every lane of the warp must call it together.
struct PassWindow {
    float cur, prev;
    MWW_D float operator()(int i) const {
        const float c = __shfl_sync(kFull, cur, i & 31), p = __shfl_sync(kFull, prev, i & 31);
        return i >= 0 ? c : p;
    }
};

// no positions: the untimed detector stores nothing beside the event, and every row's events go to the buffer
struct NoPositions {
    static constexpr bool kOffers = false;
    MWW_D void put(unsigned long long, int) const {}
};

// the warp's lanes whose `fire` is set append one event each: one atomicAdd for all of them.  Called by whole warps.  t: the
// step's index in the call, which a timed detector turns into the event's position (pos.put).  Where P::kOffers, pos.keep
// first decides whether the event goes to the buffer at all (a grouped detector offers a grouped row's event to its group)
template <typename P>
MWW_D void append_events(const DetectorArgs &a, bool fire, int row, long long step, float score, const P &pos, int t) {
    if constexpr (P::kOffers) fire = pos.keep(a, fire, row, score, t);
    const unsigned mask = __ballot_sync(kFull, fire);
    if (mask == 0) return;
    const int lane = threadIdx.x & 31;
    unsigned long long base = 0;
    if (lane == 0) base = atomicAdd(a.count, (unsigned long long)__popc(mask));
    base = __shfl_sync(kFull, base, 0);
    const unsigned long long slot = base + __popc(mask & ((1u << lane) - 1));
    if (!fire || slot >= (unsigned long long)a.capacity) return;      // past capacity: counted, not stored
    const int32_t stream = a.stream_ids ? a.stream_ids[row] : row;
    mww_event e;
    e.stream = stream; e.reserved = 0; e.step = step; e.score = score; e.pad = 0;
    a.events[slot] = e;
    a.fired[slot] = stream;
    pos.put(slot, t);
}

}  // namespace

// The update of one thread (thread form) or one warp (warp form), shared by detector_update_kernel, the timed kernel
// (mww_event_positions.cu) and the grouped one (mww_detector_groups.cu), which differ only in P.  kRowCutoff: the cutoff of
// row r is row_cutoff[r] (per-row mode); otherwise a.rule.cutoff and row_cutoff is not read.
template <bool kWarpPerRow, bool kRowCutoff, typename P>
MWW_D void detector_update_rows(const DetectorArgs &a, const float *__restrict__ probs, int n_steps, long long pitch,
                                const double *__restrict__ row_cutoff, const P &pos) {
    const DetectorRule &r = a.rule;
    if (!kWarpPerRow) {
        const long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x;
        const bool active = row < a.n_rows;                          // idle lanes stay for the ballots
        long long seen = 0;
        int cooldown = 0;
        double cutoff = r.cutoff;
        if (active) {
            seen = a.seen[row]; cooldown = a.cooldown[row];
            if (kRowCutoff) cutoff = row_cutoff[row];
        }
        RowHistory hist{a.hist + row, a.n_rows};
        for (int t = 0; t < n_steps; ++t) {
            float score = 0.f;
            bool fire = false;
            if (active) {
                fire = detector_step_at(hist, r, cutoff, seen, cooldown, probs[row * pitch + t], &score);
                ++seen;
            }
            append_events(a, fire, (int)row, seen - 1, score, pos, t);
        }
        if (active) { a.seen[row] = seen; a.cooldown[row] = cooldown; }
    } else {
        const long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
        if (row >= a.n_rows) return;                                 // whole warps leave
        const int lane = threadIdx.x & 31, w = r.window;
        const long long seen = a.seen[row];
        int cooldown = a.cooldown[row];
        const double cutoff = kRowCutoff ? row_cutoff[row] : r.cutoff;
        const float *p = probs + row * pitch;
        RowHistory hist{a.hist + row, a.n_rows};
        // the history stands in for the pass before the first: its entry j is step 32 - (w - 1) + j of that pass
        PassWindow x{0.f, lane >= 32 - (w - 1) ? hist.get(lane - (32 - (w - 1))) : 0.f};
        int n = 0;
        for (int base = 0; base < n_steps; base += 32) {
            n = min(32, n_steps - base);
            x.cur = lane < n ? p[base + lane] : 0.f;
            const float avg = detector_window_mean(x, lane, w);
            const int first = detector_first_full(seen + base, w, n);
            const unsigned candidates = __ballot_sync(kFull, lane >= first && lane < n && (double)avg > cutoff);
            const unsigned fired = detector_chain_pass(r, candidates, first, n, cooldown);
            append_events(a, (fired >> lane) & 1u, (int)row, seen + base + lane, avg, pos, base + lane);
            if (base + 32 < n_steps) x.prev = x.cur;
        }
        // new history: the last w - 1 of (old history, this call's steps), i.e. steps n - (w - 1) .. n - 1 of the last pass
        const float keep = x(lane < w - 1 ? n - (w - 1) + lane : 0);
        if (lane < w - 1) hist.set(lane, keep);
        if (lane == 0) { a.seen[row] = seen + n_steps; a.cooldown[row] = cooldown; }
    }
}

template <bool kWarpPerRow, bool kRowCutoff>
__global__ void __launch_bounds__(kThreads) detector_update_kernel(DetectorArgs a, const float *__restrict__ probs, int n_steps, long long pitch,
                                                                   const double *__restrict__ row_cutoff) {
    detector_update_rows<kWarpPerRow, kRowCutoff>(a, probs, n_steps, pitch, row_cutoff, NoPositions{});
}

// the grid of the form: a thread per row, or a warp per row from kDetectorWarpMinSteps steps on
inline unsigned update_form_blocks(const DetectorArgs &a, int n_steps) {
    const long long threads = (long long)a.n_rows * (n_steps >= kDetectorWarpMinSteps ? 32 : 1);
    return (unsigned)((threads + kThreads - 1) / kThreads);
}

// the form for a call of n_steps: thread per row below kDetectorWarpMinSteps steps, warp per row from there on
template <bool kRowCutoff>
cudaError_t launch_update_form(const DetectorArgs &a, const double *row_cutoff, const float *probs, int n_steps, long long pitch, cudaStream_t st) {
    if (n_steps <= 0 || a.n_rows <= 0) return cudaSuccess;
    if (n_steps >= kDetectorWarpMinSteps)
        detector_update_kernel<true, kRowCutoff><<<update_form_blocks(a, n_steps), kThreads, 0, st>>>(a, probs, n_steps, pitch, row_cutoff);
    else
        detector_update_kernel<false, kRowCutoff><<<update_form_blocks(a, n_steps), kThreads, 0, st>>>(a, probs, n_steps, pitch, row_cutoff);
    return cudaGetLastError();
}

}  // namespace mww
