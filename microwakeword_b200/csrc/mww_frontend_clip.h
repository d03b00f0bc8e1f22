// mww_frontend_clip.h -- the estimate chain of k1_clip_kernel (mww_frontend_clip.cu), __host__ __device__ so that
// tests/emul_frontend_clip.cc runs the very code the kernel runs.
#pragma once

#include "mww_frontend_dev.cuh"

namespace mww {

// k2_group_chain with a full group's 16 roots read before the recurrence starts.  In k2_group_chain each step's shared-memory
// load sits between two estimate updates; here the loop over frames holds only the k2_estimate_update steps, the same steps in
// the same order, so the estimates are k2_group_chain's bit for bit.  A partial group (the last of a call) takes k2_group_chain.
MWW_HD void k1_clip_chain(int ch, K1Smem &sm, int n_valid, uint32_t &est) {
    if (n_valid < kFramesPerGroup) {
        k2_group_chain(ch, sm, n_valid, est);
        return;
    }
    const uint32_t smoothing = (ch & 1) ? kOddSmoothing : kEvenSmoothing;
    uint32_t v[kFramesPerGroup];
#pragma unroll
    for (int f = 0; f < kFramesPerGroup; ++f) v[f] = sm.A[f][ch];
#pragma unroll
    for (int f = 0; f < kFramesPerGroup; ++f) {
        est = k2_estimate_update(v[f], est, smoothing);
        sm.B[f][ch] = est;
    }
}

}  // namespace mww
