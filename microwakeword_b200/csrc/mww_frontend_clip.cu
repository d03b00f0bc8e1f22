// mww_frontend_clip.cu -- the fused clip frontend (K1 + the temporal chain, features written directly), k1_clip_kernel<T, kVec>,
// for all four sample types.  It calls the phase functions of mww_frontend_dev.cuh unchanged, so the features are those of
// k1_spectral_kernel<true, 4, T> bit for bit; only the orchestration differs (DESIGN.md, K1):
//   * half-warp phase boundaries: from the window to the filterbank a frame's 16 lanes (half a warp) touch only that frame's
//     rows, so three of the six CTA-wide barriers per group are __syncwarp and a warp runs ahead instead of waiting for the
//     slowest of eight;
//   * kVec (the vector loaders apply, audio_vec_ok) is a template parameter: the aligned loop holds no per-sample loader;
//   * the estimate chain of a full group reads its 16 roots before the recurrence (k1_clip_chain, mww_frontend_clip.h), so the
//     40 chain threads, while the other six warps wait, run only the dependent k2_estimate_update steps.
// One CTA per stream, as before: persistent CTAs that walk streams (grid = the resident count) measured 7 % slower.
// A companion library of its own, libmww_frontend_clip.so, so that libmww_b200.so and libmww_g711.so keep exactly their kernels.
#include "mww_frontend.cuh"
#include "mww_frontend_clip.h"

namespace mww {

// ---- phase clocks (tools/k1_phases.py builds with -DMWW_K1_PHASE_CLOCKS; compiled out of the product): thread 0 of each CTA
// adds the clock64() cycles since its previous edge to the counter of the phase that just ended.  Thread 0 runs the estimate
// chain and waits at every CTA-wide barrier, so its timeline is the CTA's.
enum K1Phase { kPhStream, kPhTop, kPhPrefetch, kPhPass1, kPhPass2, kPhEnergy, kPhFilterbank, kPhFbBarrier, kPhChain, kPhOutputs, kK1Phases };
#ifdef MWW_K1_PHASE_CLOCKS
__device__ unsigned long long g_k1_phase_cycles[kK1Phases + 1];   // [kK1Phases]: streams completed
#define K1_PHASE_INIT long long k1_t = clock64()
#define K1_PHASE(p)                                                                                       \
    do {                                                                                                  \
        if (threadIdx.x == 0) {                                                                           \
            const long long k1_now = clock64();                                                           \
            atomicAdd(&g_k1_phase_cycles[p], (unsigned long long)(k1_now - k1_t));                        \
            k1_t = k1_now;                                                                                \
        }                                                                                                 \
    } while (0)
#else
#define K1_PHASE_INIT do {} while (0)
#define K1_PHASE(p) do {} while (0)
#endif

// group g into sm.audio[buf]: the vector loaders when kVec (asynchronous for int16 audio and the carry), else the per-sample ones
template <bool kVec, typename T>
__device__ __forceinline__ void k1_clip_load(int tid, K1Smem &sm, int buf, const int16_t *carry, int used, const T *audio, int n_samples, int g) {
    if (kVec) k1_load_audio_async(tid, sm, buf, carry, used, audio, n_samples, g * kFramesPerGroup);
    else k1_load_audio(tid, sm, buf, carry, used, audio, n_samples, g * kFramesPerGroup);
}

// grid = streams; 256 threads; 16 frames of the CTA's stream per iteration, the groups in order.
// Barrier map of one group (fl = tid >> 4 is the frame of a thread; its 16 lanes are one half of a warp):
//   top        __syncthreads  audio[buf] landed (each thread waited for its own copies) and is visible to every frame; group
//                             g-1's k2_group_outputs reads of A / B are done before this group's pass 1 and pass 2 rewrite
//                             them; audio[buf ^ 1] was last read by group g-1's pass 1, so the prefetch may overwrite it
//   pass 1 -> pass 2   __syncwarp  B[fl] (pass 1's packed points) is written and read by frame fl's lanes only
//   pass 2 -> energy   __syncwarp  A[fl] (the complex FFT) likewise; energy's B[fl] stores follow pass 2's B[fl] reads
//   energy -> filterbank __syncwarp  B[fl] (the energies) likewise; the filterbank's A[fl][0, 40) stores follow energy's
//                             A[fl] reads, and shift[fl] was written by pass 1 of the same frame
//   filterbank __syncthreads  the estimate chain (threads 0..39) reads channel ch of every frame's A row
//   chain      __syncthreads  k2_group_outputs reads every frame's estimates from B
// The next group's top barrier closes the group.  Pass 1 keeps its own __syncwarp between the lane maxima and their reads.
template <typename T, bool kVec>
__global__ void __launch_bounds__(kK1Threads, 4)
k1_clip_kernel(FrontendParams P, const int16_t *__restrict__ carry, int used, const T *__restrict__ audio, long long audio_stride,
               int n_samples, int n_frames, uint32_t *__restrict__ estimate, uint16_t *__restrict__ feat,
               long long feat_stream_stride) {
    extern __shared__ __align__(16) unsigned char k1_smem_raw[];
    K1Smem &sm = *reinterpret_cast<K1Smem *>(k1_smem_raw);
    const int tid = threadIdx.x;
    const long long s = blockIdx.x;
    K1_PHASE_INIT;
    k1_stage_lane_twiddles(tid, sm, P);
    const K1LaneShared lane_sh{&sm.lane_tw[tid & 15][0]};
    k1_stage_tables(tid, sm, P);          // visible to every thread after the first group's top barrier
    const int n_groups = (n_frames + kFramesPerGroup - 1) / kFramesPerGroup;
    const int16_t *my_carry = carry + s * kWindow;
    const T *my_audio = audio + s * audio_stride;
    uint16_t *my_feat = feat + s * feat_stream_stride;
    uint32_t est = 0;                     // thread ch < 40 carries channel ch's noise estimate across the groups
    if (tid < kNumChannels) est = estimate[s * kNumChannels + tid];
    k1_clip_load<kVec>(tid, sm, 0, my_carry, used, my_audio, n_samples, 0);
    K1_PHASE(kPhStream);
    for (int g = 0; g < n_groups; ++g) {
        const int buf = g & 1;
        cp_async_commit_and_wait_all();
        __syncthreads();
        K1_PHASE(kPhTop);
        if (g + 1 < n_groups) k1_clip_load<kVec>(tid, sm, buf ^ 1, my_carry, used, my_audio, n_samples, g + 1);
        K1_PHASE(kPhPrefetch);
        const int f0 = g * kFramesPerGroup;
        K1Pass1Ctx ctx;
        k1_window_fft1<2>(tid, sm, buf, (kHop / 2) * (tid >> 4), P, ctx);
        K1_PHASE(kPhPass1);
        __syncwarp();
        k1_fft_pass2(tid, sm, lane_sh);
        K1_PHASE(kPhPass2);
        __syncwarp();
        k1_real_energy(tid, sm, P);
        K1_PHASE(kPhEnergy);
        __syncwarp();
        k1_filterbank(tid, sm, P, &sm.A[tid >> 4][0]);    // sm.A row fl receives the frame's 40 channel values
        K1_PHASE(kPhFilterbank);
        __syncthreads();
        K1_PHASE(kPhFbBarrier);
        const int n_valid = min(kFramesPerGroup, n_frames - f0);
        if (tid < kNumChannels) k1_clip_chain(tid, sm, n_valid, est);        // estimates -> sm.B (the energies are dead)
        __syncthreads();
        K1_PHASE(kPhChain);
        k2_group_outputs(tid, sm, n_valid, my_feat + (long long)f0 * kNumChannels);
        K1_PHASE(kPhOutputs);
    }
    if (tid < kNumChannels) estimate[s * kNumChannels + tid] = est;
#ifdef MWW_K1_PHASE_CLOCKS
    if (tid == 0) atomicAdd(&g_k1_phase_cycles[kK1Phases], 1ull);
#endif
}

template <typename T>
cudaError_t launch_frontend_clip(const FrontendParams &P, const int16_t *carry, int used, const T *audio, long long audio_stride,
                                 int n_samples, int n_streams, int n_frames, uint32_t *estimate, uint16_t *feat, long long feat_stream_stride,
                                 cudaStream_t st) {
    if (n_frames <= 0 || n_streams <= 0) return cudaSuccess;
    static bool done_vec[64] = {}, done_scalar[64] = {};
    const int vec_ok = audio_vec_ok(carry, used, audio, audio_stride, n_samples);
    cudaError_t e = vec_ok ? k1_opt_in(k1_clip_kernel<T, true>, done_vec) : k1_opt_in(k1_clip_kernel<T, false>, done_scalar);
    if (e != cudaSuccess) return e;
    if (vec_ok)
        k1_clip_kernel<T, true><<<(unsigned)n_streams, kK1Threads, kK1SmemBytes, st>>>(P, carry, used, audio, audio_stride, n_samples, n_frames,
                                                                                     estimate, feat, feat_stream_stride);
    else
        k1_clip_kernel<T, false><<<(unsigned)n_streams, kK1Threads, kK1SmemBytes, st>>>(P, carry, used, audio, audio_stride, n_samples, n_frames,
                                                                                      estimate, feat, feat_stream_stride);
    return cudaGetLastError();
}

#define MWW_FRONTEND_CLIP_INSTANTIATE(T)                                                                                       \
    template cudaError_t launch_frontend_clip<T>(const FrontendParams &, const int16_t *, int, const T *, long long, int, int, int, \
                                                 uint32_t *, uint16_t *, long long, cudaStream_t);
MWW_FRONTEND_CLIP_INSTANTIATE(int16_t)
MWW_FRONTEND_CLIP_INSTANTIATE(float)
MWW_FRONTEND_CLIP_INSTANTIATE(Ulaw8)
MWW_FRONTEND_CLIP_INSTANTIATE(Alaw8)

}  // namespace mww

#ifdef MWW_K1_PHASE_CLOCKS
// phase counters of the instrumented build (tools/k1_phases.py): out[kK1Phases + 1] = cycles per phase summed over CTAs, then streams
extern "C" int mww_k1_phase_read(unsigned long long *out, int reset) {
    if (cudaDeviceSynchronize() != cudaSuccess) return 1;
    if (cudaMemcpyFromSymbol(out, mww::g_k1_phase_cycles, sizeof(mww::g_k1_phase_cycles)) != cudaSuccess) return 1;
    if (reset) {
        static const unsigned long long zero[mww::kK1Phases + 1] = {};
        if (cudaMemcpyToSymbol(mww::g_k1_phase_cycles, zero, sizeof(zero)) != cudaSuccess) return 1;
    }
    return 0;
}
#endif
