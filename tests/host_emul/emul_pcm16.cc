// tests/host_emul/emul_pcm16.cc -- TEST INFRASTRUCTURE.
//
// The float32 -> int16 sample conversion every frontend kernel applies to float audio (pcm16_from_f32 in
// microwakeword_b200/csrc/mww_frontend_dev.cuh), compiled for the CPU so that tests/test_float_audio_convert.py can check
// it against the host rule (audio_utils.to_int16) over millions of inputs.  Never used by the product.
#include <stdint.h>

#include "../../microwakeword_b200/csrc/mww_frontend_dev.cuh"

extern "C" void emul_pcm16_from_f32(const float *x, int16_t *out, long long n) {
    for (long long i = 0; i < n; ++i) out[i] = mww::pcm16_from_f32(x[i]);
}
