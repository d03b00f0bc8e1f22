// mww_resample.cuh -- the input-rate resampler kernel (definition and index math: mww_resample.h) and its launchers, included
// by the translation units that instantiate them: mww_resample.cu (the tile's streams in order, a handle with one input
// rate) and mww_resample_rates.cu (one rate's members in the tile, per-stream rates), each in a companion library of its own,
// mww_frontend_g711.cu (both, for G.711 audio) and mww_resample_mixed.cu (members with a sample format per stream).
//
// One launch per stream tile (per rate in the tile with per-stream rates) turns input-rate samples (int16, or float32
// converted by pcm16_from_f32, or G.711 decoded, on load) into 16 kHz int16 samples in scratch, which the frontend kernels then read as any
// int16 audio, and moves each stream's history forward.  Persistent CTAs: each copies the polyphase table into shared memory
// once and then takes whole streams, so the stream's history is read and rewritten by the one CTA that owns it.  Per stream
// the outputs go in chunks of kChunk: the chunk's input window (up to T - 1 samples before its first newest input, from the
// history where it reaches before the call) is staged in shared memory as int32, and each thread forms whole outputs with
// resample_output, taps and window from shared memory (CUDA cores, exact int32 products).  The kernel's Rows parameter
// (mww_resample.h) maps a CTA's stream index to its rows.
#pragma once

#include <cuda_runtime.h>

#include <algorithm>

#include "mww_frontend_dev.cuh"
#include "mww_kernels.h"
#include "mww_resample.h"

namespace mww {

constexpr int kResampleThreads = 256;
constexpr int kChunk = 1024;               // outputs per window in shared memory

// input samples a chunk of kChunk outputs reads, plus room for the history update
MWW_HD int window_cap(int T, int L, int M) { return (int)(((long long)(kChunk - 1) * M) / L) + 2 + T; }

namespace {
struct SmemWindow {
    const int32_t *xs; int lo;
    MWW_D int32_t operator()(int j) const { return xs[j - lo]; }
};
}  // namespace

// one stream of a launch, its rows x (input, samples of type T), hist and y (16 kHz output); the whole CTA runs it
template <bool kGathered, typename T>
MWW_D void resample_stream(const ResampleArgs &a, const int16_t *table, int32_t *xs, const T *x, int16_t *hist, int16_t *y) {
    if constexpr (kGathered) {
        if (a.T == 0) {                                // the identity plan (16 kHz members): no window, no history
            for (int q = threadIdx.x; q < a.n_out; q += blockDim.x) y[q] = pcm16(x[q]);
            return;
        }
    }
    for (int q0 = 0; q0 < a.n_out; q0 += kChunk) {
        const int nq = min(kChunk, a.n_out - q0);
        const int k_first = (a.t0 + q0 * a.M) / a.L;
        const int k_last = (a.t0 + (q0 + nq - 1) * a.M) / a.L;
        const int lo = k_first - (a.T - 1);
        __syncthreads();                               // the previous chunk (or stream) is done with xs
        for (int j = lo + (int)threadIdx.x; j <= k_last; j += blockDim.x)
            xs[j - lo] = j >= 0 ? (int32_t)pcm16(x[j]) : (int32_t)hist[a.H + j];
        __syncthreads();
        const SmemWindow w{xs, lo};
        for (int q = q0 + threadIdx.x; q < q0 + nq; q += blockDim.x)
            y[q] = resample_output(table, a.pitch, a.T, a.L, a.M, a.t0, q, w);
    }
    // history: the last H samples of (history, this call's input)
    __syncthreads();
    for (int j = threadIdx.x; j < a.H; j += blockDim.x) {
        const int src = a.n_in - a.H + j;
        xs[j] = src >= 0 ? (int32_t)pcm16(x[src]) : (int32_t)hist[a.H + src];
    }
    __syncthreads();
    for (int j = threadIdx.x; j < a.H; j += blockDim.x) hist[j] = (int16_t)xs[j];
}

// Rows::kMixed (MixedRows): `audio` is bytes and a.audio_stride counts bytes; each stream's row holds samples of its own
// format, which the CTA reads once and dispatches on -- a branch per stream, uniform over the CTA, none per sample.  The
// caller keeps the base and the stride multiples of 4, so float rows are aligned.
template <typename T, typename Rows>
__global__ void __launch_bounds__(kResampleThreads) resample_kernel(ResampleArgs a, const T *__restrict__ audio, int16_t *__restrict__ out, Rows rows) {
    extern __shared__ __align__(16) unsigned char smem[];
    int16_t *table = reinterpret_cast<int16_t *>(smem);
    const int table_elems = a.L * a.pitch;
    int32_t *xs = reinterpret_cast<int32_t *>(smem + ((size_t)table_elems * 2 + 15) / 16 * 16);
    for (int i = threadIdx.x; i < table_elems; i += blockDim.x) table[i] = a.table[i];
    // (the first __syncthreads of the stream loop orders the table before its first use)
    for (int s = blockIdx.x; s < a.n_streams; s += gridDim.x) {
        const T *x = audio + (size_t)rows.io(s) * a.audio_stride;
        int16_t *hist = a.hist + (size_t)rows.hist(s) * a.hist_stride;
        int16_t *y = out + (size_t)rows.io(s) * a.out_stride;
        if constexpr (Rows::kMixed) {
            switch (rows.format(s)) {
            case kFormatUlaw: resample_stream<true>(a, table, xs, reinterpret_cast<const Ulaw8 *>(x), hist, y); break;
            case kFormatAlaw: resample_stream<true>(a, table, xs, reinterpret_cast<const Alaw8 *>(x), hist, y); break;
            case kFormatF32: resample_stream<true>(a, table, xs, reinterpret_cast<const float *>(x), hist, y); break;
            default: resample_stream<true>(a, table, xs, reinterpret_cast<const int16_t *>(x), hist, y); break;
            }
        } else {
            resample_stream<Rows::kGathered>(a, table, xs, x, hist, y);
        }
    }
}

static size_t resample_smem(const ResampleArgs &a) {
    return ((size_t)a.L * a.pitch * 2 + 15) / 16 * 16 + (size_t)window_cap(a.T, a.L, a.M) * 4;
}

template <typename T, typename Rows>
cudaError_t launch_rows(const ResampleArgs &a, const T *audio, int16_t *out, Rows rows, int sm_count, cudaStream_t st) {
    if (a.n_streams <= 0 || a.n_in <= 0) return cudaSuccess;
    const size_t smem = resample_smem(a);
    static bool done[64];
    if (first_launch_on_this_device(done)) {
        cudaError_t e = cudaFuncSetAttribute(resample_kernel<T, Rows>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
        if (e != cudaSuccess) return e;
    }
    int per_sm = 0;
    cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, resample_kernel<T, Rows>, kResampleThreads, smem);
    if (e != cudaSuccess) return e;
    const int grid = std::min(a.n_streams, std::max(per_sm, 1) * sm_count);
    resample_kernel<T, Rows><<<grid, kResampleThreads, smem, st>>>(a, audio, out, rows);
    return cudaGetLastError();
}

// the launchers of mww_kernels.h, instantiated per sample type by mww_resample.cu and mww_resample_rates.cu (int16_t, float)
// and by mww_frontend_g711.cu (Ulaw8, Alaw8)
template <typename T>
cudaError_t launch_resample(const ResampleArgs &a, const T *audio, int16_t *out, int sm_count, cudaStream_t st) {
    return launch_rows(a, audio, out, TileRows{}, sm_count, st);
}
template <typename T>
cudaError_t launch_resample_members(const ResampleArgs &a, const int32_t *ids, int first, const T *audio, int16_t *out, int sm_count,
                                    cudaStream_t st) {
    return launch_rows(a, audio, out, MemberRows{ids, first}, sm_count, st);
}

}  // namespace mww
