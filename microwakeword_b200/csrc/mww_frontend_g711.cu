// mww_frontend_g711.cu -- the frontend kernels (mww_frontend.cuh) and the input-rate resampler (mww_resample.cuh) for G.711
// audio, mu-law (Ulaw8) and A-law (Alaw8): each byte is decoded to its int16 sample on load (mww_frontend_dev.cuh), so the
// window carry, the staging and every later phase are those of int16 audio.  A companion library of its own,
// libmww_g711.so, so that libmww_b200.so, libmww_resample.so and libmww_resample_rates.so keep exactly their kernels.
#include "mww_frontend.cuh"
#include "mww_resample.cuh"

namespace mww {

MWW_FRONTEND_INSTANTIATE(Ulaw8)
MWW_FRONTEND_INSTANTIATE(Alaw8)

template cudaError_t launch_resample<Ulaw8>(const ResampleArgs &, const Ulaw8 *, int16_t *, int, cudaStream_t);
template cudaError_t launch_resample<Alaw8>(const ResampleArgs &, const Alaw8 *, int16_t *, int, cudaStream_t);
template cudaError_t launch_resample_members<Ulaw8>(const ResampleArgs &, const int32_t *, int, const Ulaw8 *, int16_t *, int, cudaStream_t);
template cudaError_t launch_resample_members<Alaw8>(const ResampleArgs &, const int32_t *, int, const Alaw8 *, int16_t *, int, cudaStream_t);

}  // namespace mww
