// mww_frontend.cu -- sm_90a kernels of the batched micro-frontend (see mww_frontend_dev.cuh for the
// phase decomposition and the reference citations): the temporal kernel K2, and the kernels of mww_frontend.cuh for int16
// and float32 audio.
#include <cuda_runtime.h>
#include <stdlib.h>

#include "mww_frontend.cuh"

namespace mww {

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

bool frontend_clip_fuses(int n_streams, int n_frames, int sm_count) {
    // one CTA per stream walks the stream's groups in order; below ~12 CTAs per SM's worth of streams the frames of a stream
    // are spread over several CTAs instead (grid.y > 1) and the temporal chain stays a separate kernel
    return n_frames > 8 && (long long)n_streams >= (long long)sm_count * 3 * 4;
}

bool frontend_fusable(int used, int n_samples, int n_frames) {
    const int new_used = used + n_samples - n_frames * kHop;
    return n_frames >= 1 && n_frames <= 8 && new_used >= 0 && new_used <= 2 * kHop;
}

cudaError_t launch_k2(const FrontendParams &P, const uint32_t *vin, int n_streams, int n_frames, uint32_t *estimate,
                      uint16_t *feat, long long feat_stream_stride, cudaStream_t st) {
    if (n_frames <= 0 || n_streams <= 0) return cudaSuccess;
    const long long total = (long long)n_streams * kNumChannels;
    const unsigned blocks = (unsigned)((total + 255) / 256);
    k2_temporal_kernel<<<blocks, 256, 0, st>>>(P, vin, n_streams, n_frames, estimate, feat, feat_stream_stride);
    return cudaGetLastError();
}

MWW_FRONTEND_INSTANTIATE(int16_t)
MWW_FRONTEND_INSTANTIATE(float)

}  // namespace mww
