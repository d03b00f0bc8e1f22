// mww_frontend.cu -- sm_90a kernels of the batched micro-frontend (see mww_frontend_dev.cuh for the
// phase decomposition and the reference citations).
#include <cuda_runtime.h>
#include <stdlib.h>

#include "mww_frontend_dev.cuh"
#include "mww_kernels.h"

namespace mww {

// 16-byte async copies global -> shared (LDGSTS): the next group's audio lands while this one is computed
__device__ __forceinline__ void cp_async16(void *smem_dst, const void *gmem_src) {
    const unsigned dst = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(gmem_src));
}
__device__ __forceinline__ void cp_async_commit_and_wait_all() {
    asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory");
}

// 8 caller samples -> 16 bytes of int16 staging.  int16 audio: one asynchronous copy.  float32 audio: two float4 loads
// through registers, converted (pcm16_from_f32) and stored; the copy itself is then synchronous, the rest of the kernel is
// unchanged.
__device__ __forceinline__ void stage8(int16_t *dst, const int16_t *src) { cp_async16(dst, src); }
__device__ __forceinline__ void stage8(int16_t *dst, const float *src) {
    const float4 a = reinterpret_cast<const float4 *>(src)[0], b = reinterpret_cast<const float4 *>(src)[1];
    *reinterpret_cast<uint4 *>(dst) = make_uint4(pack16(pcm16_from_f32(a.x), pcm16_from_f32(a.y)), pack16(pcm16_from_f32(a.z), pcm16_from_f32(a.w)),
                                                 pack16(pcm16_from_f32(b.x), pcm16_from_f32(b.y)), pack16(pcm16_from_f32(b.z), pcm16_from_f32(b.w)));
}

// vectorised variant of k1_load_audio: valid when `used`, `n_samples` and the row pitch are multiples of 8
// samples and both base pointers are 16-byte aligned, so no 8-sample vector straddles a source boundary
template <typename T>
__device__ __forceinline__ void k1_load_audio_async(int tid, K1Smem &sm, int buf, const int16_t *carry, int used,
                                                    const T *audio, int n_samples, int f0) {
    const int base = kHop * f0;
    for (int v = tid; v < kGroupSamples / 8; v += kK1Threads) {
        const int vi = base + 8 * v;
        int16_t *dst = &sm.audio[buf][8 * v];
        if (vi < used) cp_async16(dst, carry + vi);
        else if (vi - used < n_samples) stage8(dst, audio + (vi - used));
        else *reinterpret_cast<uint4 *>(dst) = make_uint4(0, 0, 0, 0);
    }
}

// vectorised variant of k1_packed_load_audio (same alignment conditions): 8 samples per 16-byte copy instead of one
// 2-byte load + an integer division per sample
template <typename T>
__device__ __forceinline__ void k1_packed_load_audio_async(int tid, K1Smem &sm, const int16_t *carry, int used, const T *audio,
                                                           long long audio_stride, int n_samples, long long s0, int n_streams, int spc, int fps) {
    const int span8 = (fps + 2) * (kHop / 8), used8 = used / 8, n8 = n_samples / 8;
    int16_t *dst0 = &sm.audio[0][0];
    for (int i = tid; i < spc * span8; i += kK1Threads) {
        const int sl = i / span8, v8 = i - sl * span8;
        int16_t *dst = dst0 + 8 * i;
        const long long s = s0 + sl;
        if (s < n_streams && v8 < used8) cp_async16(dst, carry + s * kWindow + 8 * v8);
        else if (s < n_streams && v8 - used8 < n8) stage8(dst, audio + s * audio_stride + 8 * (v8 - used8));
        else *reinterpret_cast<uint4 *>(dst) = make_uint4(0, 0, 0, 0);
    }
}

// K1: grid = (streams, group_chunks); 256 threads; 16 frames of one stream per iteration.
// kFuseK2 (grid.y == 1: the CTA walks all of its stream's groups in order): the temporal chain -- noise estimate, PCAN, log --
// runs from shared memory right behind the filterbank and the kernel writes the uint16 feature rows itself; no V round trip
// through HBM, no K2 launch, no scratch buffer.
// kOcc = CTAs per SM the kernel is compiled for: 3 keeps the per-lane FFT twiddles in registers (80 registers), 4 reads them
// from shared memory (64 registers).
// T = sample type of the caller's audio (int16_t or float) in this and every kernel below that reads it.
template <bool kFuseK2, int kOcc, typename T>
__global__ void __launch_bounds__(kK1Threads, kOcc)
k1_spectral_kernel(FrontendParams P, const int16_t *__restrict__ carry, int used,
                   const T *__restrict__ audio, long long audio_stride, int n_samples, int n_frames,
                   int groups_per_block, int vec_ok, uint32_t *__restrict__ vout, uint32_t *__restrict__ estimate,
                   uint16_t *__restrict__ feat, long long feat_stream_stride) {
    extern __shared__ __align__(16) unsigned char k1_smem_raw[];
    K1Smem &sm = *reinterpret_cast<K1Smem *>(k1_smem_raw);
    const int tid = threadIdx.x;
    const long long s = blockIdx.x;
    K1Lane lane;
    if (kOcc <= 3) k1_lane_init(tid, P, lane);
    else k1_stage_lane_twiddles(tid, sm, P);
    const K1LaneShared lane_sh{&sm.lane_tw[tid & 15][0]};
    k1_stage_tables(tid, sm, P);

    const int n_groups = (n_frames + kFramesPerGroup - 1) / kFramesPerGroup;
    const int g_begin = blockIdx.y * groups_per_block;
    const int g_end = min(g_begin + groups_per_block, n_groups);
    const int16_t *my_carry = carry + s * kWindow;
    const T *my_audio = audio + s * audio_stride;
    uint32_t est = 0;                          // fused: thread ch < 40 carries channel ch's noise estimate across the groups
    if (kFuseK2 && tid < kNumChannels) est = estimate[s * kNumChannels + tid];
    if (g_begin < g_end) {
        if (vec_ok) k1_load_audio_async(tid, sm, 0, my_carry, used, my_audio, n_samples, g_begin * kFramesPerGroup);
        else k1_load_audio(tid, sm, 0, my_carry, used, my_audio, n_samples, g_begin * kFramesPerGroup);
    }
    for (int g = g_begin; g < g_end; ++g) {
        const int buf = (g - g_begin) & 1;
        cp_async_commit_and_wait_all();
        __syncthreads();                       // audio[buf] visible; everyone is done with the previous group
        if (g + 1 < g_end) {                   // prefetch: audio[buf^1] was last read two barriers ago
            if (vec_ok) k1_load_audio_async(tid, sm, buf ^ 1, my_carry, used, my_audio, n_samples, (g + 1) * kFramesPerGroup);
            else k1_load_audio(tid, sm, buf ^ 1, my_carry, used, my_audio, n_samples, (g + 1) * kFramesPerGroup);
        }
        const int f0 = g * kFramesPerGroup;
        K1Pass1Ctx ctx;
        k1_window_fft1<2>(tid, sm, buf, (kHop / 2) * (tid >> 4), P, ctx);
        __syncthreads();
        if (kOcc <= 3) k1_fft_pass2(tid, sm, lane); else k1_fft_pass2(tid, sm, lane_sh);
        __syncthreads();
        k1_real_energy(tid, sm, P);
        __syncthreads();
        const int f = f0 + (tid >> 4);
        if (!kFuseK2) {
            k1_filterbank(tid, sm, P, f < n_frames ? vout + (s * n_frames + f) * kNumChannels : nullptr);
            // hazards: the next iteration's top barrier orders filterbank's reads of B/shift before the next
            // window_fft1 rewrites them; A is rewritten only after two more barriers (DESIGN.md, K1)
        } else {
            // sm.A is free from here on (real_energy consumed it): row fl receives the frame's 40 channel values
            k1_filterbank(tid, sm, P, &sm.A[tid >> 4][0]);
            __syncthreads();
            const int n_valid = min(kFramesPerGroup, n_frames - f0);
            if (tid < kNumChannels) k2_group_chain(tid, sm, n_valid, est);       // estimates -> sm.B (the energies are dead)
            __syncthreads();
            k2_group_outputs(tid, sm, n_valid, feat + s * feat_stream_stride + (long long)f0 * kNumChannels);
            // hazards: the next iteration's top barrier orders these reads of A / B before window_fft1 rewrites B
        }
    }
    if (kFuseK2 && tid < kNumChannels) estimate[s * kNumChannels + tid] = est;
}

// Run-time hop variant of the fused clip kernel (any even hop <= 480 samples, i.e. window_step up to 30 ms): one CTA per
// stream, groups of k1_hop_frames_per_group(hop) frames, single-buffered audio staging.  Used only when the handle's hop is
// not the 10 ms every shipped model uses; the 10 ms kernels above stay specialised.  72 registers (launched with 256 threads):
// three CTAs per SM, as the shared memory allows.  nvcc rejects __launch_bounds__ and __maxnreg__ on the same kernel, so the
// block size is not declared here; launch_frontend_hop is its only launcher and always uses kK1Threads.
template <typename T>
__global__ void __maxnreg__(72)
k1_spectral_hop_kernel(FrontendParams P, const int16_t *__restrict__ carry, int used, const T *__restrict__ audio,
                       long long audio_stride, int n_samples, int n_frames, int hop, uint32_t *__restrict__ estimate,
                       uint16_t *__restrict__ feat, long long feat_stream_stride) {
    extern __shared__ __align__(16) unsigned char k1_smem_raw[];
    K1Smem &sm = *reinterpret_cast<K1Smem *>(k1_smem_raw);
    const int tid = threadIdx.x;
    const long long s = blockIdx.x;
    K1Lane lane;
    k1_lane_init(tid, P, lane);
    k1_stage_tables(tid, sm, P);
    const int fpg = k1_hop_frames_per_group(hop);
    const int n_groups = (n_frames + fpg - 1) / fpg;
    const int16_t *my_carry = carry + s * kWindow;
    const T *my_audio = audio + s * audio_stride;
    uint32_t est = 0;
    if (tid < kNumChannels) est = estimate[s * kNumChannels + tid];
    for (int g = 0; g < n_groups; ++g) {
        const int f0 = g * fpg;
        __syncthreads();                       // everyone is done with the previous group's staging area, A and B
        k1_hop_load_audio(tid, sm, my_carry, used, my_audio, n_samples, hop * f0, (fpg - 1) * hop + kWindow);
        __syncthreads();
        K1Pass1Ctx ctx;
        k1_window_fft1<2>(tid, sm, 0, k1_hop_pair_base(tid >> 4, hop, fpg), P, ctx);
        __syncthreads();
        k1_fft_pass2(tid, sm, lane);
        __syncthreads();
        k1_real_energy(tid, sm, P);
        __syncthreads();
        k1_filterbank(tid, sm, P, &sm.A[tid >> 4][0]);
        __syncthreads();
        const int n_valid = min(fpg, n_frames - f0);
        if (tid < kNumChannels) k2_group_chain(tid, sm, n_valid, est);
        __syncthreads();
        k2_group_outputs(tid, sm, n_valid, feat + s * feat_stream_stride + (long long)f0 * kNumChannels);
    }
    if (tid < kNumChannels) estimate[s * kNumChannels + tid] = est;
}

// K1 for short calls (n_frames <= 8, e.g. the three frames of a 30 ms live step): one CTA = `spc` streams x `fps`
// frames, so the 16 frame slots stay (almost) full instead of serving 3 of 16.
template <typename T>
__global__ void __launch_bounds__(kK1Threads, 3)
k1_spectral_packed_kernel(FrontendParams P, const int16_t *__restrict__ carry, int used,
                          const T *__restrict__ audio, long long audio_stride, int n_samples, int n_streams, int fps, int spc,
                          int vec_ok, uint32_t *__restrict__ vout) {
    extern __shared__ __align__(16) unsigned char k1_smem_raw[];
    K1Smem &sm = *reinterpret_cast<K1Smem *>(k1_smem_raw);
    const int tid = threadIdx.x;
    const long long s0 = (long long)blockIdx.x * spc;
    K1Lane lane;
    k1_lane_init(tid, P, lane);
    k1_stage_tables(tid, sm, P);
    if (vec_ok) {
        k1_packed_load_audio_async(tid, sm, carry, used, audio, audio_stride, n_samples, s0, n_streams, spc, fps);
        cp_async_commit_and_wait_all();
    } else {
        k1_packed_load_audio(tid, sm, carry, used, audio, audio_stride, n_samples, s0, n_streams, spc, fps);
    }
    __syncthreads();
    const int fl = tid >> 4;
    K1Pass1Ctx ctx;
    k1_window_fft1<2>(tid, sm, 0, k1_packed_pair_base(fl < spc * fps ? fl : 0, fps), P, ctx);
    __syncthreads();
    k1_fft_pass2(tid, sm, lane);
    __syncthreads();
    k1_real_energy(tid, sm, P);
    __syncthreads();
    const long long s = s0 + fl / fps;
    const bool active = fl < spc * fps && s < n_streams;
    k1_filterbank(tid, sm, P, active ? vout + (s * fps + fl % fps) * kNumChannels : nullptr);
}

// Whole frontend of a short call in ONE launch: packed K1, then -- all frames of a CTA's streams being resident -- the
// K2 temporal chain (noise reduction -> PCAN -> log) straight from shared memory, then the carry update from the staged
// audio.  Saves the V round trip through HBM and two launches per live step.  Requires new_used <= 2 hops (the staged
// span ends 2 hops after the last frame's start) -- the launcher checks.
template <typename T>
__global__ void __launch_bounds__(kK1Threads, 3)
k1k2_packed_kernel(FrontendParams P, int16_t *__restrict__ carry, int used, const T *__restrict__ audio,
                   long long audio_stride, int n_samples, int n_streams, int fps, int spc, int vec_ok, uint32_t *__restrict__ estimate,
                   uint16_t *__restrict__ feat, long long feat_stream_stride, int new_used) {
    extern __shared__ __align__(16) unsigned char k1_smem_raw[];
    K1Smem &sm = *reinterpret_cast<K1Smem *>(k1_smem_raw);
    const int tid = threadIdx.x;
    const long long s0 = (long long)blockIdx.x * spc;
    K1Lane lane;
    k1_lane_init(tid, P, lane);
    k1_stage_tables(tid, sm, P);
    if (vec_ok) {
        k1_packed_load_audio_async(tid, sm, carry, used, audio, audio_stride, n_samples, s0, n_streams, spc, fps);
        cp_async_commit_and_wait_all();
    } else {
        k1_packed_load_audio(tid, sm, carry, used, audio, audio_stride, n_samples, s0, n_streams, spc, fps);
    }
    __syncthreads();
    const int fl = tid >> 4;
    K1Pass1Ctx ctx;
    k1_window_fft1<2>(tid, sm, 0, k1_packed_pair_base(fl < spc * fps ? fl : 0, fps), P, ctx);
    __syncthreads();
    k1_fft_pass2(tid, sm, lane);
    __syncthreads();
    k1_real_energy(tid, sm, P);
    __syncthreads();
    // sm.A is free from here on: row fl receives the frame's 40 channel energies
    k1_filterbank(tid, sm, P, fl < spc * fps ? &sm.A[fl][0] : nullptr);
    __syncthreads();
    for (int t = tid; t < spc * kNumChannels; t += kK1Threads) {        // up to 12 streams x 40 channels per CTA
        const int sl = t / kNumChannels, ch = t - sl * kNumChannels;
        const long long s = s0 + sl;
        if (s < n_streams) {
            const uint32_t smoothing = (ch & 1) ? kOddSmoothing : kEvenSmoothing;
            uint32_t est = estimate[s * kNumChannels + ch];
            uint16_t *out = feat + s * feat_stream_stride + ch;
            for (int f = 0; f < fps; ++f) out[(long long)f * kNumChannels] = k2_channel_step(sm.A[sl * fps + f][ch], est, smoothing, sm.gain_lut, sm.log_lut);
            estimate[s * kNumChannels + ch] = est;
        }
    }
    // carry: samples [consumed, consumed + new_used) of (old carry ++ audio) are staged at span offset `consumed`
    const int span = (fps + 2) * kHop, consumed = fps * kHop;
    const int16_t *staged = &sm.audio[0][0];
    if (vec_ok) {
        for (int i = tid; i < spc * (kWindow / 8); i += kK1Threads) {
            const int sl = i / (kWindow / 8), v8 = i - sl * (kWindow / 8);
            if (s0 + sl >= n_streams) continue;
            uint4 v = make_uint4(0, 0, 0, 0);
            if (8 * v8 < new_used) v = *reinterpret_cast<const uint4 *>(staged + sl * span + consumed + 8 * v8);
            *reinterpret_cast<uint4 *>(carry + (s0 + sl) * kWindow + 8 * v8) = v;
        }
    } else {
        for (int i = tid; i < spc * kWindow; i += kK1Threads) {
            const int sl = i / kWindow, k = i - sl * kWindow;
            if (s0 + sl >= n_streams) continue;
            carry[(s0 + sl) * kWindow + k] = k < new_used ? staged[sl * span + consumed + k] : (int16_t)0;
        }
    }
}

// K2: one thread per (stream, channel); frames are scanned in order, noise estimate kept in a register.
__global__ void __launch_bounds__(256)
k2_temporal_kernel(FrontendParams P, const uint32_t *__restrict__ vin, int n_streams, int n_frames,
                   uint32_t *__restrict__ estimate, uint16_t *__restrict__ feat, long long feat_stream_stride) {
    __shared__ int16_t gain_lut[128];
    __shared__ uint16_t log_lut[132];
    for (int i = threadIdx.x; i < 128; i += blockDim.x) gain_lut[i] = P.gain_lut[i];
    for (int i = threadIdx.x; i < 132; i += blockDim.x) log_lut[i] = P.log_lut[i];
    __syncthreads();
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)n_streams * kNumChannels) return;
    const long long s = idx / kNumChannels;
    const int ch = (int)(idx - s * kNumChannels);
    const uint32_t smoothing = (ch & 1) ? kOddSmoothing : kEvenSmoothing;
    uint32_t est = estimate[idx];
    const uint32_t *v = vin + s * (long long)n_frames * kNumChannels + ch;
    uint16_t *out = feat + s * feat_stream_stride + ch;
    int f = 0;
    for (; f + 4 <= n_frames; f += 4) {
        uint32_t x[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) x[q] = __ldcs(v + (long long)(f + q) * kNumChannels);
#pragma unroll
        for (int q = 0; q < 4; ++q) out[(long long)(f + q) * kNumChannels] = k2_channel_step(x[q], est, smoothing, gain_lut, log_lut);
    }
    for (; f < n_frames; ++f) out[(long long)f * kNumChannels] = k2_channel_step(v[(long long)f * kNumChannels], est, smoothing, gain_lut, log_lut);
    estimate[idx] = est;
}

// carry update: keep the samples that did not complete a hop (one CTA of 128 threads per stream); float audio is
// converted, so the carry always holds int16 samples
template <typename T>
__global__ void __launch_bounds__(128)
carry_update_kernel(int16_t *__restrict__ carry, int used, const T *__restrict__ audio, long long audio_stride,
                    int n_samples, int consumed, int new_used) {
    const long long s = blockIdx.x;
    int16_t *c = carry + s * kWindow;
    const T *a = audio + s * audio_stride;
    int16_t tmp[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const int i = threadIdx.x + 128 * q;
        int16_t val = 0;
        if (i < new_used) {
            const int vi = consumed + i;
            val = vi < used ? c[vi] : pcm16(a[vi - used]);
        }
        tmp[q] = val;
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const int i = threadIdx.x + 128 * q;
        if (i < kWindow) c[i] = tmp[q];
    }
}

// ---------------------------------------------------------------------------------------------
// launchers

namespace {
// K1Smem is above the 48 KB static limit: dynamic shared memory, opted in per kernel and per device
template <typename K>
cudaError_t k1_opt_in(K kernel, bool (&done)[64]) {
    if (!first_launch_on_this_device(done)) return cudaSuccess;
    return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kK1SmemBytes);
}
// the 16-byte loaders (k1_load_audio_async) apply: 8-sample vectors never straddle the carry / audio boundary or a row end,
// and both sources are 16-byte aligned (8 int16 samples = one cp.async, 8 float samples = two float4 loads)
template <typename T>
int audio_vec_ok(const int16_t *carry, int used, const T *audio, long long audio_stride, int n_samples) {
    return (used % 8 == 0) && (n_samples % 8 == 0) && (audio_stride % 8 == 0) &&
           (reinterpret_cast<uintptr_t>(audio) % 16 == 0) && (reinterpret_cast<uintptr_t>(carry) % 16 == 0);
}
}  // namespace

bool frontend_clip_fuses(int n_streams, int n_frames, int sm_count) {
    // one CTA per stream walks the stream's groups in order; below ~12 CTAs per SM's worth of streams the frames of a stream
    // are spread over several CTAs instead (grid.y > 1) and the temporal chain stays a separate kernel
    return n_frames > 8 && (long long)n_streams >= (long long)sm_count * 3 * 4;
}

template <typename T>
cudaError_t launch_k1(const FrontendParams &P, const int16_t *carry, int used, const T *audio,
                      long long audio_stride, int n_samples, int n_streams, int n_frames, uint32_t *vout, int sm_count,
                      cudaStream_t st) {
    if (n_frames <= 0 || n_streams <= 0) return cudaSuccess;
    const int vec_ok = audio_vec_ok(carry, used, audio, audio_stride, n_samples);
    if (n_frames <= 8 && n_streams >= 2) {
        static bool done[64] = {};
        cudaError_t e = k1_opt_in(k1_spectral_packed_kernel<T>, done);
        if (e != cudaSuccess) return e;
        const int spc = k1_packed_streams(n_frames);
        const unsigned grid = (unsigned)((n_streams + spc - 1) / spc);
        k1_spectral_packed_kernel<T><<<grid, kK1Threads, kK1SmemBytes, st>>>(P, carry, used, audio, audio_stride, n_samples, n_streams, n_frames, spc, vec_ok, vout);
        return cudaGetLastError();
    }
    static bool done[64] = {};
    cudaError_t e = k1_opt_in(k1_spectral_kernel<false, 3, T>, done);
    if (e != cudaSuccess) return e;
    const int n_groups = (n_frames + kFramesPerGroup - 1) / kFramesPerGroup;
    // enough CTAs to fill the chip a few times over, but keep per-CTA setup amortised when streams abound
    int chunks = 1;
    const long long want = (long long)sm_count * 3 * 4;
    if (n_streams < want) chunks = (int)min((long long)n_groups, (want + n_streams - 1) / n_streams);
    const int gpb = (n_groups + chunks - 1) / chunks;
    chunks = (n_groups + gpb - 1) / gpb;
    dim3 grid((unsigned)n_streams, (unsigned)chunks);
    k1_spectral_kernel<false, 3, T><<<grid, kK1Threads, kK1SmemBytes, st>>>(P, carry, used, audio, audio_stride, n_samples, n_frames, gpb, vec_ok, vout,
                                                                         nullptr, nullptr, 0);
    return cudaGetLastError();
}

template <typename T>
cudaError_t launch_frontend_clip_fused(const FrontendParams &P, const int16_t *carry, int used, const T *audio, long long audio_stride,
                                       int n_samples, int n_streams, int n_frames, uint32_t *estimate, uint16_t *feat, long long feat_stream_stride,
                                       cudaStream_t st) {
    if (n_frames <= 0 || n_streams <= 0) return cudaSuccess;
    static bool done3[64] = {}, done4[64] = {};
    static const int occ = getenv("MWW_K1_OCC") ? atoi(getenv("MWW_K1_OCC")) : 4;
    cudaError_t e = occ == 3 ? k1_opt_in(k1_spectral_kernel<true, 3, T>, done3) : k1_opt_in(k1_spectral_kernel<true, 4, T>, done4);
    if (e != cudaSuccess) return e;
    const int vec_ok = audio_vec_ok(carry, used, audio, audio_stride, n_samples);
    const int n_groups = (n_frames + kFramesPerGroup - 1) / kFramesPerGroup;
    dim3 grid((unsigned)n_streams, 1u);
    if (occ == 3)
        k1_spectral_kernel<true, 3, T><<<grid, kK1Threads, kK1SmemBytes, st>>>(P, carry, used, audio, audio_stride, n_samples, n_frames, n_groups, vec_ok,
                                                                               nullptr, estimate, feat, feat_stream_stride);
    else
        k1_spectral_kernel<true, 4, T><<<grid, kK1Threads, kK1SmemBytes, st>>>(P, carry, used, audio, audio_stride, n_samples, n_frames, n_groups, vec_ok,
                                                                               nullptr, estimate, feat, feat_stream_stride);
    return cudaGetLastError();
}

template <typename T>
cudaError_t launch_frontend_hop(const FrontendParams &P, const int16_t *carry, int used, const T *audio, long long audio_stride,
                                int n_samples, int n_streams, int n_frames, int hop, uint32_t *estimate, uint16_t *feat,
                                long long feat_stream_stride, cudaStream_t st) {
    if (n_frames <= 0 || n_streams <= 0) return cudaSuccess;
    static bool done[64] = {};
    cudaError_t e = k1_opt_in(k1_spectral_hop_kernel<T>, done);
    if (e != cudaSuccess) return e;
    k1_spectral_hop_kernel<T><<<(unsigned)n_streams, kK1Threads, kK1SmemBytes, st>>>(P, carry, used, audio, audio_stride, n_samples, n_frames, hop,
                                                                                    estimate, feat, feat_stream_stride);
    return cudaGetLastError();
}

bool frontend_fusable(int used, int n_samples, int n_frames) {
    const int new_used = used + n_samples - n_frames * kHop;
    return n_frames >= 1 && n_frames <= 8 && new_used >= 0 && new_used <= 2 * kHop;
}

template <typename T>
cudaError_t launch_frontend_fused(const FrontendParams &P, int16_t *carry, int used, const T *audio,
                                  long long audio_stride, int n_samples, int n_streams, int n_frames, uint32_t *estimate, uint16_t *feat,
                                  long long feat_stream_stride, cudaStream_t st) {
    if (n_streams <= 0) return cudaSuccess;
    static bool done[64] = {};
    cudaError_t e = k1_opt_in(k1k2_packed_kernel<T>, done);
    if (e != cudaSuccess) return e;
    const int vec_ok = audio_vec_ok(carry, used, audio, audio_stride, n_samples);
    const int spc = k1_packed_streams(n_frames);
    const unsigned grid = (unsigned)((n_streams + spc - 1) / spc);
    k1k2_packed_kernel<T><<<grid, kK1Threads, kK1SmemBytes, st>>>(P, carry, used, audio, audio_stride, n_samples, n_streams, n_frames, spc, vec_ok,
                                                                  estimate, feat, feat_stream_stride, used + n_samples - n_frames * kHop);
    return cudaGetLastError();
}

cudaError_t launch_k2(const FrontendParams &P, const uint32_t *vin, int n_streams, int n_frames, uint32_t *estimate,
                      uint16_t *feat, long long feat_stream_stride, cudaStream_t st) {
    if (n_frames <= 0 || n_streams <= 0) return cudaSuccess;
    const long long total = (long long)n_streams * kNumChannels;
    const unsigned blocks = (unsigned)((total + 255) / 256);
    k2_temporal_kernel<<<blocks, 256, 0, st>>>(P, vin, n_streams, n_frames, estimate, feat, feat_stream_stride);
    return cudaGetLastError();
}

template <typename T>
cudaError_t launch_carry_update(int16_t *carry, int used, const T *audio, long long audio_stride, int n_samples,
                                int n_streams, int consumed, int new_used, cudaStream_t st) {
    if (n_streams <= 0) return cudaSuccess;
    carry_update_kernel<T><<<(unsigned)n_streams, 128, 0, st>>>(carry, used, audio, audio_stride, n_samples, consumed, new_used);
    return cudaGetLastError();
}

// the two sample types the C-ABI accepts on device (mww_features / mww_predict_clip and their _f32 forms)
#define MWW_FRONTEND_INSTANTIATE(T)                                                                                            \
    template cudaError_t launch_k1<T>(const FrontendParams &, const int16_t *, int, const T *, long long, int, int, int, uint32_t *, \
                                      int, cudaStream_t);                                                                      \
    template cudaError_t launch_frontend_clip_fused<T>(const FrontendParams &, const int16_t *, int, const T *, long long, int, int, \
                                                       int, uint32_t *, uint16_t *, long long, cudaStream_t);                 \
    template cudaError_t launch_frontend_hop<T>(const FrontendParams &, const int16_t *, int, const T *, long long, int, int, int, \
                                                int, uint32_t *, uint16_t *, long long, cudaStream_t);                        \
    template cudaError_t launch_frontend_fused<T>(const FrontendParams &, int16_t *, int, const T *, long long, int, int, int,   \
                                                  uint32_t *, uint16_t *, long long, cudaStream_t);                           \
    template cudaError_t launch_carry_update<T>(int16_t *, int, const T *, long long, int, int, int, int, cudaStream_t);
MWW_FRONTEND_INSTANTIATE(int16_t)
MWW_FRONTEND_INSTANTIATE(float)
#undef MWW_FRONTEND_INSTANTIATE

}  // namespace mww
