// tests/host_emul/emul_g711.cc -- TEST INFRASTRUCTURE.
//
// The G.711 decode every frontend and resampler kernel applies to mu-law and A-law audio (pcm16 of Ulaw8 / Alaw8 in
// microwakeword_b200/csrc/mww_frontend_dev.cuh), compiled for the CPU so that tests/test_g711.py can check all 256 codes of
// each law against the rule in include/mww.h and against Python's audioop.  Never used by the product.
#include <stdint.h>

#include "../../microwakeword_b200/csrc/mww_frontend_dev.cuh"

extern "C" void emul_g711_decode(int law, const uint8_t *codes, int16_t *out, long long n) {
    for (long long i = 0; i < n; ++i) out[i] = law == 1 ? mww::pcm16(mww::Ulaw8{codes[i]}) : mww::pcm16(mww::Alaw8{codes[i]});
}
