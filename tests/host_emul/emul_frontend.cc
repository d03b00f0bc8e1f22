// tests/host_emul/emul_frontend.cc -- TEST INFRASTRUCTURE.
//
// Executes the product's frontend PHASE functions (microwakeword_b200/csrc/mww_frontend_dev.cuh --
// the very code the sm_90a kernels run) on the CPU, thread by thread with barriers modelled as
// "finish the phase for all 256 threads", so index math / bit-exactness can be validated against
// the oracle in the GPU-less authoring container.  Never used by the product.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../microwakeword_b200/csrc/mww_frontend_dev.cuh"

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

int emul_tables(int16_t *window480, int16_t *bin_weight257, int16_t *bin_unweight257, int16_t *chan_start42,
                int16_t *gain_lut125, uint16_t *log_lut129, int16_t *tw512, int16_t *super256, int32_t *info8) {
    ensure_tables();
    const HostTables &t = g_tables;
    memcpy(window480, t.window, sizeof t.window);
    memcpy(bin_weight257, t.bin_weight, sizeof t.bin_weight);
    memcpy(bin_unweight257, t.bin_unweight, sizeof t.bin_unweight);
    memcpy(chan_start42, t.chan_start, sizeof t.chan_start);
    memcpy(gain_lut125, t.gain_lut, 125 * sizeof(int16_t));
    memcpy(log_lut129, t.log_lut, 129 * sizeof(uint16_t));
    for (int k = 0; k < 256; ++k) { tw512[2 * k] = (int16_t)unpack_lo(t.tw[k]); tw512[2 * k + 1] = (int16_t)unpack_hi(t.tw[k]); }
    for (int k = 0; k < 128; ++k) { super256[2 * k] = (int16_t)unpack_lo(t.super_tw[k]); super256[2 * k + 1] = (int16_t)unpack_hi(t.super_tw[k]); }
    info8[0] = t.start_index; info8[1] = t.end_index; info8[2] = t.ok;
    info8[3] = (int)t.fb_coef.size();
    for (int s = 0; s < kFbSlots; ++s) if (t.fb_slot_len[s] != kFbLen[s]) return -1;
    for (int s = 0; s < kFbSlots; ++s) info8[4 + s] = t.fb_slot_len[s];
    return 0;
}

uint32_t emul_isqrt64_round(uint64_t x) { return isqrt64_round(x); }
uint32_t emul_isqrt64_round_fast(uint64_t x) { return isqrt64_round_fast(x); }
// first index where the FP64 fast path and the integer routine disagree, -1 if none (bulk fuzz without ctypes overhead)
long long emul_isqrt_fast_mismatch(const uint64_t *x, long long n) {
    for (long long i = 0; i < n; ++i) if (isqrt64_round_fast(x[i]) != isqrt64_round(x[i])) return i;
    return -1;
}

// Mirrors mww_features(): streams advance in lockstep; returns the number of feature rows per stream.
int emul_features(const int16_t *audio, int n_streams, int n_samples, int16_t *carry, int used, uint32_t *estimate,
                  uint16_t *feat, int max_rows, int *new_used_out) {
    ensure_tables();
    const int total = used + n_samples;
    const int n_frames = total >= kWindow ? (total - kWindow) / kHop + 1 : 0;
    const int consumed = n_frames * kHop;
    const int new_used = total - consumed;
    std::vector<uint32_t> v((size_t)n_streams * (n_frames > 0 ? n_frames : 1) * kNumChannels);
    K1Smem *sm = new K1Smem;
    std::vector<K1Lane> lanes(kK1Threads);
    const int n_groups = (n_frames + kFramesPerGroup - 1) / kFramesPerGroup;
    if (n_frames > 0 && n_frames <= 8 && n_streams >= 2) {
        // packed mapping (mirrors launch_k1): several streams per CTA
        const int fps = n_frames, spc = k1_packed_streams(fps);
        for (long long s0 = 0; s0 < n_streams; s0 += spc) {
            memset(sm, 0xA5, sizeof *sm);
            for (int tid = 0; tid < kK1Threads; ++tid) k1_lane_init(tid, g_params, lanes[tid]);
            for (int tid = 0; tid < kK1Threads; ++tid) k1_stage_tables(tid, *sm, g_params);
            for (int tid = 0; tid < kK1Threads; ++tid) k1_packed_load_audio(tid, *sm, carry, used, audio, n_samples, n_samples, s0, n_streams, spc, fps);
            std::vector<K1Pass1Ctx> ctx(kK1Threads);
            for (int part = 0; part < 2; ++part)
                for (int tid = 0; tid < kK1Threads; ++tid) {
                    const int fl = tid >> 4, pb = k1_packed_pair_base(fl < spc * fps ? fl : 0, fps);
                    if (part == 0) k1_window_fft1<0>(tid, *sm, 0, pb, g_params, ctx[tid]); else k1_window_fft1<1>(tid, *sm, 0, pb, g_params, ctx[tid]);
                }
            for (int tid = 0; tid < kK1Threads; ++tid) k1_fft_pass2(tid, *sm, lanes[tid]);
            for (int tid = 0; tid < kK1Threads; ++tid) k1_real_energy(tid, *sm, g_params);
            for (int tid = 0; tid < kK1Threads; ++tid) {
                const int fl = tid >> 4;
                const long long s = s0 + fl / fps;
                const bool active = fl < spc * fps && s < n_streams;
                k1_filterbank(tid, *sm, g_params, active ? &v[((size_t)s * fps + fl % fps) * kNumChannels] : nullptr);
            }
        }
    } else
    for (int s = 0; s < n_streams; ++s) {
        memset(sm, 0xA5, sizeof *sm);   // poison: phases must not depend on stale shared memory
        for (int tid = 0; tid < kK1Threads; ++tid) k1_lane_init(tid, g_params, lanes[tid]);
        for (int tid = 0; tid < kK1Threads; ++tid) k1_stage_tables(tid, *sm, g_params);
        const int16_t *my_carry = carry + (size_t)s * kWindow;
        const int16_t *my_audio = audio + (size_t)s * n_samples;
        for (int g = 0; g < n_groups; ++g) {
            const int f0 = g * kFramesPerGroup;
            const int buf = g & 1;
            for (int tid = 0; tid < kK1Threads; ++tid) k1_load_audio(tid, *sm, buf, my_carry, used, my_audio, n_samples, f0);
            std::vector<K1Pass1Ctx> ctx(kK1Threads);
            for (int tid = 0; tid < kK1Threads; ++tid) k1_window_fft1<0>(tid, *sm, buf, (kHop / 2) * (tid >> 4), g_params, ctx[tid]);   // half-warp exchange between
            for (int tid = 0; tid < kK1Threads; ++tid) k1_window_fft1<1>(tid, *sm, buf, (kHop / 2) * (tid >> 4), g_params, ctx[tid]);
            for (int tid = 0; tid < kK1Threads; ++tid) k1_fft_pass2(tid, *sm, lanes[tid]);
            for (int tid = 0; tid < kK1Threads; ++tid) k1_real_energy(tid, *sm, g_params);
            for (int tid = 0; tid < kK1Threads; ++tid) {
                const int f = f0 + (tid >> 4);
                k1_filterbank(tid, *sm, g_params, f < n_frames ? &v[((size_t)s * n_frames + f) * kNumChannels] : nullptr);
            }
        }
    }
    delete sm;
    for (int s = 0; s < n_streams; ++s)
        for (int ch = 0; ch < kNumChannels; ++ch) {
            uint32_t est = estimate[(size_t)s * kNumChannels + ch];
            const uint32_t smoothing = (ch & 1) ? kOddSmoothing : kEvenSmoothing;
            for (int f = 0; f < n_frames && f < max_rows; ++f)
                feat[((size_t)s * max_rows + f) * kNumChannels + ch] =
                    k2_channel_step(v[((size_t)s * n_frames + f) * kNumChannels + ch], est, smoothing, g_tables.gain_lut, g_tables.log_lut);
            estimate[(size_t)s * kNumChannels + ch] = est;
        }
    // carry update
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

// Mirrors the fused clip kernel (k1_spectral_kernel<true>): one "CTA" per stream walks the groups in order; after the
// filterbank the temporal chain runs from shared memory (k2_group_chain on threads 0..39, then k2_group_outputs on all 256).
// `order` 0 = ascending thread order inside every phase, 1 = descending (an intra-phase race would show as a difference).
int emul_features_fused(const int16_t *audio, int n_streams, int n_samples, int16_t *carry, int used, uint32_t *estimate,
                        uint16_t *feat, int max_rows, int *new_used_out, int order) {
    ensure_tables();
    const int total = used + n_samples;
    const int n_frames = total >= kWindow ? (total - kWindow) / kHop + 1 : 0;
    const int consumed = n_frames * kHop;
    const int new_used = total - consumed;
    if (n_frames > max_rows) return -1;
    K1Smem *sm = new K1Smem;
    std::vector<K1Lane> lanes(kK1Threads);
    const int n_groups = (n_frames + kFramesPerGroup - 1) / kFramesPerGroup;
    auto T = [&](int i) { return order ? kK1Threads - 1 - i : i; };
    for (int s = 0; s < n_streams; ++s) {
        memset(sm, 0xA5, sizeof *sm);
        for (int i = 0; i < kK1Threads; ++i) k1_stage_lane_twiddles(T(i), *sm, g_params);     // the 4-CTA/SM variant: twiddles from shared memory
        for (int i = 0; i < kK1Threads; ++i) k1_stage_tables(T(i), *sm, g_params);
        const int16_t *my_carry = carry + (size_t)s * kWindow;
        const int16_t *my_audio = audio + (size_t)s * n_samples;
        uint32_t est[kNumChannels];
        for (int ch = 0; ch < kNumChannels; ++ch) est[ch] = estimate[(size_t)s * kNumChannels + ch];
        for (int g = 0; g < n_groups; ++g) {
            const int f0 = g * kFramesPerGroup;
            const int buf = g & 1;
            for (int i = 0; i < kK1Threads; ++i) k1_load_audio(T(i), *sm, buf, my_carry, used, my_audio, n_samples, f0);
            std::vector<K1Pass1Ctx> ctx(kK1Threads);
            for (int i = 0; i < kK1Threads; ++i) k1_window_fft1<0>(T(i), *sm, buf, (kHop / 2) * (T(i) >> 4), g_params, ctx[T(i)]);
            for (int i = 0; i < kK1Threads; ++i) k1_window_fft1<1>(T(i), *sm, buf, (kHop / 2) * (T(i) >> 4), g_params, ctx[T(i)]);
            for (int i = 0; i < kK1Threads; ++i) k1_fft_pass2(T(i), *sm, K1LaneShared{&sm->lane_tw[T(i) & 15][0]});
            for (int i = 0; i < kK1Threads; ++i) k1_real_energy(T(i), *sm, g_params);
            for (int i = 0; i < kK1Threads; ++i) k1_filterbank(T(i), *sm, g_params, &sm->A[T(i) >> 4][0]);
            const int n_valid = n_frames - f0 < kFramesPerGroup ? n_frames - f0 : kFramesPerGroup;
            for (int i = 0; i < kK1Threads; ++i) if (T(i) < kNumChannels) k2_group_chain(T(i), *sm, n_valid, est[T(i)]);
            for (int i = 0; i < kK1Threads; ++i) k2_group_outputs(T(i), *sm, n_valid, feat + ((size_t)s * max_rows + f0) * kNumChannels);
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

// Mirrors k1_spectral_hop_kernel (run-time window step): groups of k1_hop_frames_per_group(hop) frames, single staging area.
int emul_features_hop(const int16_t *audio, int n_streams, int n_samples, int16_t *carry, int used, uint32_t *estimate,
                      uint16_t *feat, int max_rows, int *new_used_out, int hop) {
    ensure_tables();
    const int total = used + n_samples;
    const int n_frames = total >= kWindow ? (total - kWindow) / hop + 1 : 0;
    const int consumed = n_frames * hop;
    const int new_used = total - consumed;
    if (n_frames > max_rows || new_used < 0 || new_used >= kWindow) return -1;
    K1Smem *sm = new K1Smem;
    std::vector<K1Lane> lanes(kK1Threads);
    const int fpg = k1_hop_frames_per_group(hop);
    const int n_groups = (n_frames + fpg - 1) / fpg;
    for (int s = 0; s < n_streams; ++s) {
        memset(sm, 0xA5, sizeof *sm);
        for (int tid = 0; tid < kK1Threads; ++tid) k1_lane_init(tid, g_params, lanes[tid]);
        for (int tid = 0; tid < kK1Threads; ++tid) k1_stage_tables(tid, *sm, g_params);
        const int16_t *my_carry = carry + (size_t)s * kWindow;
        const int16_t *my_audio = audio + (size_t)s * n_samples;
        uint32_t est[kNumChannels];
        for (int ch = 0; ch < kNumChannels; ++ch) est[ch] = estimate[(size_t)s * kNumChannels + ch];
        for (int g = 0; g < n_groups; ++g) {
            const int f0 = g * fpg;
            for (int tid = 0; tid < kK1Threads; ++tid) k1_hop_load_audio(tid, *sm, my_carry, used, my_audio, n_samples, hop * f0, (fpg - 1) * hop + kWindow);
            std::vector<K1Pass1Ctx> ctx(kK1Threads);
            for (int tid = 0; tid < kK1Threads; ++tid) k1_window_fft1<0>(tid, *sm, 0, k1_hop_pair_base(tid >> 4, hop, fpg), g_params, ctx[tid]);
            for (int tid = 0; tid < kK1Threads; ++tid) k1_window_fft1<1>(tid, *sm, 0, k1_hop_pair_base(tid >> 4, hop, fpg), g_params, ctx[tid]);
            for (int tid = 0; tid < kK1Threads; ++tid) k1_fft_pass2(tid, *sm, lanes[tid]);
            for (int tid = 0; tid < kK1Threads; ++tid) k1_real_energy(tid, *sm, g_params);
            for (int tid = 0; tid < kK1Threads; ++tid) k1_filterbank(tid, *sm, g_params, &sm->A[tid >> 4][0]);
            const int n_valid = n_frames - f0 < fpg ? n_frames - f0 : fpg;
            for (int tid = 0; tid < kNumChannels; ++tid) k2_group_chain(tid, *sm, n_valid, est[tid]);
            for (int tid = 0; tid < kK1Threads; ++tid) k2_group_outputs(tid, *sm, n_valid, feat + ((size_t)s * max_rows + f0) * kNumChannels);
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

// filterbank schedule for the conflict-freedom test: slots16x4x4 = (ch, word0, n, coef_off) per lane and slot
void emul_fb_schedule(int16_t *slots16x4x4, int32_t *coef800) {
    ensure_tables();
    for (int l = 0; l < kFbLanes; ++l)
        for (int s = 0; s < kFbSlots; ++s) {
            const FbSlot &q = g_tables.fb_slots[l][s];
            int16_t *o = slots16x4x4 + (l * kFbSlots + s) * 4;
            o[0] = q.ch; o[1] = q.word0; o[2] = q.n; o[3] = q.coef_off;
        }
    for (int i = 0; i < kFbCoefWords; ++i) coef800[i] = g_tables.fb_coef[i];
}

}  // extern "C"
