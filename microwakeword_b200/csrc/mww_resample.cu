// mww_resample.cu -- the input-rate resampler (kernel: mww_resample.cuh; definition and index math: mww_resample.h) on the
// streams of a tile in order, for a handle with one input rate.  Its companion mww_resample_rates.cu instantiates the same
// kernel on one rate's members of a tile (per-stream rates) in a library of its own.
#include "mww_resample.cuh"

namespace mww {

template cudaError_t launch_resample<int16_t>(const ResampleArgs &, const int16_t *, int16_t *, int, cudaStream_t);
template cudaError_t launch_resample<float>(const ResampleArgs &, const float *, int16_t *, int, cudaStream_t);

}  // namespace mww
