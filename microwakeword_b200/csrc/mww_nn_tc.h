// mww_nn_tc.h -- launcher of the wgmma clip kernel (mww_nn_tc.cu) and the host-side weight preparation it needs.
#pragma once

#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <vector>

#include "mww_nn_dev.cuh"

namespace mww {

// Device pointers to the 3xTF32-split weights in tensor-core slot layout (build_tc_weights): K cut into slots of 32 values, a slot =
// hi plane [N rows][128 B, 128-byte swizzle] followed by the lo plane.  fc: first conv, K = 200 (7 slots), N = 32; pw[i]: 1x1 of block i.
struct TcWeights {
    const unsigned char *fc;
    const unsigned char *pw[4];
};

constexpr int kTcMinSteps = 16;     // shorter calls stay on the mma.sync kernel (a 128-step tile would be mostly padding)

// host: split + lay out; `blob` is what gets uploaded, offsets[0] = first conv, offsets[1 + i] = block i (256-byte aligned)
void build_tc_weights(const float *w0, const float *const pw[4], std::vector<unsigned char> *blob, size_t offsets[5]);

cudaError_t launch_nn_f32_tc(const NnWeightsF32 &W, const TcWeights &TW, float *state, float *pend, int n_pend, const uint16_t *rows,
                             long long rows_stream_stride, int n_rows, float *probs, long long probs_stream_stride, int n_streams, int sm_count,
                             cudaStream_t st);

}  // namespace mww
