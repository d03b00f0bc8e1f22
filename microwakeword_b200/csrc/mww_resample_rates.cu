// mww_resample_rates.cu -- the input-rate resampler (kernel: mww_resample.cuh) on the members of one rate in a stream tile,
// for a handle with per-stream rates (mww_set_stream_rates): one launch per rate present in the tile.  Its own companion
// library, so that libmww_resample.so keeps exactly the kernels a handle with one input rate runs.
#include "mww_resample.cuh"

namespace mww {

template cudaError_t launch_resample_members<int16_t>(const ResampleArgs &, const int32_t *, int, const int16_t *, int16_t *, int, cudaStream_t);
template cudaError_t launch_resample_members<float>(const ResampleArgs &, const int32_t *, int, const float *, int16_t *, int, cudaStream_t);

}  // namespace mww
