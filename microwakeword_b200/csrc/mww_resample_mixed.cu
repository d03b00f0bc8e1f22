// mww_resample_mixed.cu -- the input-rate resampler (kernel: mww_resample.cuh) on the members of one rate in a stream tile
// whose rows each hold their own sample format (mww_set_stream_formats, the _mixed entry points): int16, float32, mu-law or
// A-law, decoded on load by the body of that format.  Its own companion library, so that libmww_resample_rates.so and
// libmww_g711.so keep exactly their kernels.
#include "mww_resample.cuh"

namespace mww {

cudaError_t launch_resample_mixed(const ResampleArgs &a, const int32_t *ids, int first, const uint8_t *formats, const Mixed8 *audio,
                                  int16_t *out, int sm_count, cudaStream_t st) {
    return launch_rows(a, audio, out, MixedRows{ids, first, formats}, sm_count, st);
}

}  // namespace mww
