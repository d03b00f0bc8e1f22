// mww_tables.h -- host-built constant tables of the fixed-point micro-frontend, in the packed
// layouts the sm_90a kernels consume.  Replaces the table construction that
// pymicro_features.MicroFrontend() performs when the reference instantiates it at
// microwakeword/audio/audio_utils.py:52 (window / KissFFT twiddles / mel filterbank weights /
// PCAN gain LUT / log LUT; algorithm per SURVEY.md Appendix B).
#pragma once

#include <stdint.h>

#include <vector>

#include "mww_common.h"

namespace mww {

constexpr int kFbLanes = 16;       // lanes that cooperate on one frame
constexpr int kFbSlots = 4;        // max channels one lane accumulates
// Shared-memory layout of the span coefficients: int32 (no unpack instruction before the 32x32->64 multiply-add),
// [slot][lane][stride] with strides of 2 x odd words so that the 16 lanes of a frame hit 16 distinct bank PAIRS with
// their 64-bit loads (stride / 2 odd => lane * stride / 2 is a permutation mod 16).
constexpr int kFbCoefStride[3] = {30, 14, 6};                  // words per lane and slot (trip counts 28, 12, 6 below)
constexpr int kFbCoefWords = 16 * (30 + 14 + 6);               // 800 int32 = 3 200 B
// Energy of FFT bin k is stored at word k + kEnergyOffset of the frame's row, and every span starts at an EVEN word
// (zero coefficients in front where the true first bin is odd or the start was moved down): the energies are fetched
// two per 64-bit load, and the start words of the 16 lanes of a slot are chosen (bipartite matching at table-build
// time, mww_tables.cc) so that (start / 2) mod 16 is a permutation -- no shared-memory bank conflict in the mel
// accumulation (the natural layout puts the lanes of these loads on the same banks).
constexpr int kEnergyOffset = 1;
// Trip counts of the balanced filterbank schedule (mww_tables.cc LPT assignment), padded to even so the
// Q12 coefficients can be fetched two per 32-bit load.  mww_create verifies the table builder agrees.
constexpr int kFbLen[kFbSlots] = {28, 12, 6, 0};
MWW_HD constexpr int fb_len(int s) { return s == 0 ? 28 : (s == 1 ? 12 : (s == 2 ? 6 : 0)); }
static_assert(fb_len(0) == kFbLen[0] && fb_len(1) == kFbLen[1] && fb_len(2) == kFbLen[2] && fb_len(3) == kFbLen[3], "fb_len");

struct FbSlot {
    int16_t ch;        // output channel 0..39, -1 = unused slot
    int16_t word0;     // first (even) word of the span inside the frame's energy row (bin + kEnergyOffset - leading zeros)
    int16_t n;         // bins in the span (informational)
    int16_t coef_off;  // even offset into fb_coef, in int32 words (the span is zero padded to the slot's uniform length)
};

// Tables passed BY VALUE as a kernel parameter (lives in the constant bank; uniform reads are free).
struct FrontendParams {
    const uint32_t *win_pairs;   // [240] window coefficients, two Q12 int16 per word
    const uint32_t *tw;          // [256] exp(-2*pi*i*k/256) Q15, (re | im << 16)
    const uint32_t *super_tw;    // [128] real-FFT post-pass twiddles, same packing
    const int32_t *fb_coef;      // [kFbCoefWords] filterbank span coefficients (Q12 as int32), zero padded
    const FbSlot *fb_slots;      // [16][kFbSlots]
    const int16_t *gain_lut;     // [128] PCAN wide-dynamic-function LUT (125 used)
    const uint16_t *log_lut;     // [132] log2 correction LUT (129 used)
    int16_t tw2[9][2];           // stage-2 twiddles tw[16k], tw[32k], tw[48k] for k = 1..3
    int32_t fb_slot_len[kFbSlots];
};

struct HostTables {
    // packed, kernel-facing
    uint32_t win_pairs[240];
    uint32_t tw[256];
    uint32_t super_tw[128];
    std::vector<int32_t> fb_coef;
    FbSlot fb_slots[kFbLanes][kFbSlots];
    int32_t fb_slot_len[kFbSlots];
    int16_t gain_lut[128];
    uint16_t log_lut[132];
    int16_t tw2[9][2];
    // logical, test-facing
    int16_t window[480];
    int16_t bin_channel[257], bin_weight[257], bin_unweight[257];
    int16_t chan_start[42];
    int start_index, end_index;
    bool ok;
};

// noise-reduction / PCAN / log scalars (SURVEY.md Appendix B steps 7-9)
constexpr int kSmoothingBits = 10;
constexpr uint32_t kEvenSmoothing = 409;       // int(0.025 * 2^14)
constexpr uint32_t kOddSmoothing = 983;        // int(0.06  * 2^14)
constexpr uint32_t kMinSignalRemaining = 819;  // int(0.05  * 2^14)
constexpr int kNoiseBits = 14;
constexpr int kPcanSnrShift = 6;               // gain_bits 21 - correction 3 - snr bits 12
constexpr int kLogCorrectionBits = 3;          // msb(512) - 1 - 12/2
constexpr int kLogScaleShift = 6;

void build_host_tables(HostTables *t);

}  // namespace mww
