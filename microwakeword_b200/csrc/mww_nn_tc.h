// mww_nn_tc.h -- launcher of the wgmma clip kernel (mww_nn_tc.cu) and the host-side weight preparation it needs.
#pragma once

#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <vector>

#include "mww_nn_dev.cuh"
#include "mww_nn_tc_prep.h"

namespace mww {

// Device pointers to the 3xTF32-split weights in tensor-core slot layout (build_tc_weights): K cut into slots of 32 values, a slot =
// hi plane [N rows][128 B, 128-byte swizzle] followed by the lo plane.  fc: first conv, K = 200 (7 slots), N = 32; pw[i]: 1x1 of block i.
// fc16: the first conv's weights x 0.0390625 x 2^s_fc as fp16 hi / lo operands (tc_layout_f16): K = 200 cut into 4 slots of 64, a
// slot = hi plane [32 rows][128 B] followed by the lo plane; its epilogue undoes the scale with the exact multiply fc_out = 2^-s_fc.
struct TcWeights {
    const unsigned char *fc;
    const unsigned char *pw[4];
    const unsigned char *fc16;
    float fc_out;
};

constexpr int kTcMinSteps = 16;     // shorter calls stay on the mma.sync kernel (a 128-step tile would be mostly padding)

// host: split + lay out; `blob` is what gets uploaded, offsets[0] = first conv, offsets[1 + i] = block i (256-byte aligned);
// with f16 (from tc_f16_scales, ok) the first conv's fp16 operands follow at offsets[5]
void build_tc_weights(const float *w0, const float *const pw[4], const TcF16Scales *f16, std::vector<unsigned char> *blob,
                      size_t offsets[6]);

// f16: the kernel whose first conv takes the integer features as fp16 A operands (TW.fc16; the feature rows and the state's
// first-conv ring and pending rows must be integer features <= 2048 -- x 0.0390625 for the latter two); otherwise 3xTF32 throughout
cudaError_t launch_nn_f32_tc(const NnWeightsF32 &W, const TcWeights &TW, bool f16, float *state, float *pend, int n_pend, const uint16_t *rows,
                             long long rows_stream_stride, int n_rows, float *probs, long long probs_stream_stride, int n_streams, int sm_count,
                             cudaStream_t st);

}  // namespace mww
