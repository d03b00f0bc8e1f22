// tests/emul_frontend_clip.cc -- TEST INFRASTRUCTURE: the group schedule of the fused clip kernel k1_clip_kernel
// (microwakeword_b200/csrc/mww_frontend_clip.cu) on the CPU, built with g++ by tests/test_frontend_clip_kernel.py against the
// product's phase functions (mww_frontend_dev.cuh, the code the kernel runs).  One CTA per stream walks the groups in order.
//
//   * The next group's audio is loaded into the other buffer right after the top barrier, before this group's pass 1, as the
//     kernel issues it.
//   * Between the top barrier and the filterbank barrier only __syncwarp separates the phases, so the emulation runs one warp
//     (two frames) through window + FFT pass 1, pass 2, the post-pass and the filterbank before the next warp starts: a phase
//     that read another warp's rows would read the previous group's values (or the poison) and the features would differ.
//     `order` 1 reverses the warp order and the thread order inside every phase.
//   * The estimate chain (k1_clip_chain, mww_frontend_clip.h) and the outputs run between CTA-wide barriers, as in the kernel.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../microwakeword_b200/csrc/mww_frontend_clip.h"

using namespace mww;

namespace {
HostTables g_tables;
FrontendParams g_params;
bool g_ready = false;

void ensure_tables() {
    if (g_ready) return;
    build_host_tables(&g_tables);
    g_params.win_pairs = g_tables.win_pairs;
    g_params.tw = g_tables.tw;
    g_params.super_tw = g_tables.super_tw;
    g_params.fb_coef = g_tables.fb_coef.data();
    g_params.fb_slots = &g_tables.fb_slots[0][0];
    g_params.gain_lut = g_tables.gain_lut;
    g_params.log_lut = g_tables.log_lut;
    memcpy(g_params.tw2, g_tables.tw2, sizeof g_params.tw2);
    memcpy(g_params.fb_slot_len, g_tables.fb_slot_len, sizeof g_params.fb_slot_len);
    g_ready = true;
}
}  // namespace

extern "C" {

// One clip call of n_streams int16 streams; returns the feature rows per stream (features in feat [n_streams][max_rows][40]),
// -1 when they do not fit.  Carry, used and estimate advance as the product's call does (the carry update is its own kernel).
int emul_clip_features(const int16_t *audio, int n_streams, int n_samples, int16_t *carry, int used, uint32_t *estimate,
                       uint16_t *feat, int max_rows, int *new_used_out, int order) {
    ensure_tables();
    const int total = used + n_samples;
    const int n_frames = total >= kWindow ? (total - kWindow) / kHop + 1 : 0;
    const int consumed = n_frames * kHop;
    const int new_used = total - consumed;
    if (n_frames > max_rows) return -1;
    const int n_groups = (n_frames + kFramesPerGroup - 1) / kFramesPerGroup;
    constexpr int kWarps = kK1Threads / 32;
    auto T = [&](int i, int n) { return order ? n - 1 - i : i; };
    K1Smem *sm = new K1Smem;
    std::vector<K1Pass1Ctx> ctx(kK1Threads);
    for (int s = 0; s < n_streams; ++s) {
        const int16_t *my_carry = carry + (size_t)s * kWindow;
        const int16_t *my_audio = audio + (size_t)s * n_samples;
        auto load = [&](int buf, int g) {
            for (int i = 0; i < kK1Threads; ++i) k1_load_audio(T(i, kK1Threads), *sm, buf, my_carry, used, my_audio, n_samples, g * kFramesPerGroup);
        };
        memset(sm, 0xA5, sizeof *sm);   // poison: phases must not depend on stale shared memory
        for (int i = 0; i < kK1Threads; ++i) k1_stage_lane_twiddles(T(i, kK1Threads), *sm, g_params);
        for (int i = 0; i < kK1Threads; ++i) k1_stage_tables(T(i, kK1Threads), *sm, g_params);
        uint32_t est[kNumChannels];
        for (int ch = 0; ch < kNumChannels; ++ch) est[ch] = estimate[(size_t)s * kNumChannels + ch];
        if (n_groups > 0) load(0, 0);
        for (int g = 0; g < n_groups; ++g) {
            const int buf = g & 1;
            // top barrier
            if (g + 1 < n_groups) load(buf ^ 1, g + 1);
            for (int wi = 0; wi < kWarps; ++wi) {
                const int w = T(wi, kWarps);
                auto lane = [&](int i) { return 32 * w + T(i, 32); };
                for (int i = 0; i < 32; ++i) k1_window_fft1<0>(lane(i), *sm, buf, (kHop / 2) * (lane(i) >> 4), g_params, ctx[lane(i)]);
                for (int i = 0; i < 32; ++i) k1_window_fft1<1>(lane(i), *sm, buf, (kHop / 2) * (lane(i) >> 4), g_params, ctx[lane(i)]);
                // __syncwarp
                for (int i = 0; i < 32; ++i) k1_fft_pass2(lane(i), *sm, K1LaneShared{&sm->lane_tw[lane(i) & 15][0]});
                // __syncwarp
                for (int i = 0; i < 32; ++i) k1_real_energy(lane(i), *sm, g_params);
                // __syncwarp
                for (int i = 0; i < 32; ++i) k1_filterbank(lane(i), *sm, g_params, &sm->A[lane(i) >> 4][0]);
            }
            // filterbank barrier
            const int f0 = g * kFramesPerGroup;
            const int n_valid = n_frames - f0 < kFramesPerGroup ? n_frames - f0 : kFramesPerGroup;
            for (int i = 0; i < kK1Threads; ++i) if (T(i, kK1Threads) < kNumChannels) k1_clip_chain(T(i, kK1Threads), *sm, n_valid, est[T(i, kK1Threads)]);
            // chain barrier
            for (int i = 0; i < kK1Threads; ++i)
                k2_group_outputs(T(i, kK1Threads), *sm, n_valid, feat + ((size_t)s * max_rows + f0) * kNumChannels);
        }
        for (int ch = 0; ch < kNumChannels; ++ch) estimate[(size_t)s * kNumChannels + ch] = est[ch];
    }
    delete sm;
    for (int s = 0; s < n_streams; ++s) {
        int16_t tmp[kWindow] = {0};
        int16_t *c = carry + (size_t)s * kWindow;
        for (int i = 0; i < new_used; ++i) {
            const int vi = consumed + i;
            tmp[i] = vi < used ? c[vi] : audio[(size_t)s * n_samples + (vi - used)];
        }
        memcpy(c, tmp, sizeof tmp);
    }
    if (new_used_out) *new_used_out = new_used;
    return n_frames;
}

int emul_k1_smem_bytes() { return kK1SmemBytes; }

}  // extern "C"
