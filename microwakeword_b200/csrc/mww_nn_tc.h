// mww_nn_tc.h -- launcher of the wgmma clip kernel (mww_nn_tc.cu); its weight operands: mww_nn_tc_prep.h.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "mww_nn_dev.cuh"
#include "mww_nn_tc_prep.h"

namespace mww {

constexpr int kTcMinSteps = 16;     // shorter calls stay on the mma.sync kernel (a 128-step tile would be mostly padding)

// f16: the kernel whose first conv takes the integer features as fp16 A operands (TW.fc16; the feature rows and the state's
// first-conv ring and pending rows must be integer features <= 2048 -- x 0.0390625 for the latter two); otherwise 3xTF32 throughout
cudaError_t launch_nn_f32_tc(const NnWeightsF32 &W, const TcWeights &TW, bool f16, float *state, float *pend, int n_pend, const uint16_t *rows,
                             long long rows_stream_stride, int n_rows, float *probs, long long probs_stream_stride, int n_streams, int sm_count,
                             cudaStream_t st);

}  // namespace mww
