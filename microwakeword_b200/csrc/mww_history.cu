// mww_history.cu -- the two kernels of the audio history (mww_set_audio_history; ring layout and index math: mww_history.h).
// Pure data movement, one work unit per thread over streams x units in a grid-stride loop, so that one 480-sample live call
// at 65 536 streams (3.9 M vector units) spreads over every SM.  A companion library of its own, libmww_history.so, so that
// libmww_b200.so keeps exactly the kernels a handle without a history runs.
#include <algorithm>

#include "mww_history.h"
#include "mww_kernels.h"

namespace mww {

namespace {

constexpr int kHistoryThreads = 256;

// 8 caller samples -> 8 int16 samples packed in 16 bytes: one 16-byte load for int16, two float4 loads converted with
// pcm16_from_f32 for float32, one 8-byte load decoded for the G.711 types
__device__ __forceinline__ uint4 load8(const int16_t *src) { return *reinterpret_cast<const uint4 *>(src); }
__device__ __forceinline__ uint4 load8(const float *src) {
    const float4 a = reinterpret_cast<const float4 *>(src)[0], b = reinterpret_cast<const float4 *>(src)[1];
    return make_uint4(pack16(pcm16_from_f32(a.x), pcm16_from_f32(a.y)), pack16(pcm16_from_f32(a.z), pcm16_from_f32(a.w)),
                      pack16(pcm16_from_f32(b.x), pcm16_from_f32(b.y)), pack16(pcm16_from_f32(b.z), pcm16_from_f32(b.w)));
}
template <typename G>
__device__ __forceinline__ uint4 load8_g711(const G *src) {
    const uint2 c = *reinterpret_cast<const uint2 *>(src);
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const uint32_t word = i < 2 ? c.x : c.y, sh = 16 * (i & 1);
        w[i] = pack16(pcm16(G{(uint8_t)(word >> sh)}), pcm16(G{(uint8_t)(word >> (sh + 8))}));
    }
    return make_uint4(w[0], w[1], w[2], w[3]);
}
__device__ __forceinline__ uint4 load8(const Ulaw8 *src) { return load8_g711(src); }
__device__ __forceinline__ uint4 load8(const Alaw8 *src) { return load8_g711(src); }

// the last p.m samples of a call of every stream of the tile -> their ring slots.  vec: units of 8 samples (16-byte stores,
// the loads of load8), else one sample per unit.
template <typename T>
__global__ void __launch_bounds__(kHistoryThreads)
history_append_kernel(int16_t *__restrict__ ring, int C, const T *__restrict__ audio, long long audio_stride, HistoryAppend p, int n_streams,
                      int vec) {
    const int units = vec ? p.m / 8 : p.m;
    const long long total = (long long)n_streams * units;
    for (long long i = (long long)blockIdx.x * kHistoryThreads + threadIdx.x; i < total; i += (long long)gridDim.x * kHistoryThreads) {
        const long long s = i / units;
        const int u = (int)(i - s * units);
        int16_t *row = ring + s * C;
        const T *src = audio + s * audio_stride;
        if (vec) *reinterpret_cast<uint4 *>(row + history_slot(p.slot0, 8 * u, C)) = load8(src + p.src0 + 8 * u);
        else history_append_one(row, src, p, u, C);
    }
}

// n rows of n_samples: row i is the last n_samples of stream ids[i] (zeros for an id outside [0, n_streams)), entry k from
// slot history_slot(slot0, k, C).  vec: units of 8 entries, 16-byte loads and stores.
__global__ void __launch_bounds__(kHistoryThreads)
history_read_kernel(const int16_t *__restrict__ ring, int C, const int32_t *__restrict__ ids, int n, int n_streams, int slot0, int n_samples,
                    int16_t *__restrict__ out, long long out_stride, int vec) {
    const int units = vec ? n_samples / 8 : n_samples;
    const long long total = (long long)n * units;
    for (long long i = (long long)blockIdx.x * kHistoryThreads + threadIdx.x; i < total; i += (long long)gridDim.x * kHistoryThreads) {
        const long long r = i / units;
        const int u = (int)(i - r * units);
        const int id = ids[r];
        int16_t *dst = out + r * out_stride;
        if (vec) {
            uint4 v = make_uint4(0, 0, 0, 0);
            if (id >= 0 && id < n_streams) v = *reinterpret_cast<const uint4 *>(ring + (long long)id * C + history_slot(slot0, 8 * u, C));
            *reinterpret_cast<uint4 *>(dst + 8 * u) = v;
        } else {
            dst[u] = history_read_one(ring, C, id, n_streams, slot0, u);
        }
    }
}

unsigned history_blocks(long long total, int sm_count) {
    return (unsigned)std::max<long long>(1, std::min<long long>((total + kHistoryThreads - 1) / kHistoryThreads, (long long)sm_count * 16));
}

}  // namespace

// The vector form applies when history_append_vec_shape holds and the caller's audio is aligned for load8: 16 bytes for
// int16 and float32, 8 bytes for the 1-byte G.711 samples -- the condition audio_vec_ok states for the frontend's loaders.
// Rows of the ring start on 16 bytes (C % 8 == 0, cudaMalloc alignment).
template <typename T>
int history_append_vec_ok(const HistoryAppend &p, const T *audio, long long audio_stride) {
    constexpr uintptr_t kAlign = sizeof(T) == 1 ? 8 : 16;
    return history_append_vec_shape(p, audio_stride) && reinterpret_cast<uintptr_t>(audio) % kAlign == 0;
}

template <typename T>
cudaError_t launch_history_append(int16_t *ring, int C, long long seen, const T *audio, long long audio_stride, int n16, int n_streams,
                                  int sm_count, cudaStream_t st) {
    if (n16 <= 0 || n_streams <= 0 || C <= 0) return cudaSuccess;
    const HistoryAppend p = history_append_plan(seen, n16, C);
    const int vec = history_append_vec_ok(p, audio, audio_stride);
    const long long total = (long long)n_streams * (vec ? p.m / 8 : p.m);
    history_append_kernel<T><<<history_blocks(total, sm_count), kHistoryThreads, 0, st>>>(ring, C, audio, audio_stride, p, n_streams, vec);
    return cudaGetLastError();
}

cudaError_t launch_history_read(const int16_t *ring, int C, long long seen, const int32_t *ids, int n, int n_streams, int n_samples, int16_t *out,
                                long long out_stride, int sm_count, cudaStream_t st) {
    if (n <= 0 || n_samples <= 0) return cudaSuccess;
    const int slot0 = history_read_slot0(seen, n_samples, C);
    const int vec = history_read_vec_shape(slot0, n_samples, out_stride) && reinterpret_cast<uintptr_t>(out) % 16 == 0;
    const long long total = (long long)n * (vec ? n_samples / 8 : n_samples);
    history_read_kernel<<<history_blocks(total, sm_count), kHistoryThreads, 0, st>>>(ring, C, ids, n, n_streams, slot0, n_samples, out, out_stride,
                                                                                     vec);
    return cudaGetLastError();
}

template cudaError_t launch_history_append<int16_t>(int16_t *, int, long long, const int16_t *, long long, int, int, int, cudaStream_t);
template cudaError_t launch_history_append<float>(int16_t *, int, long long, const float *, long long, int, int, int, cudaStream_t);
template cudaError_t launch_history_append<Ulaw8>(int16_t *, int, long long, const Ulaw8 *, long long, int, int, int, cudaStream_t);
template cudaError_t launch_history_append<Alaw8>(int16_t *, int, long long, const Alaw8 *, long long, int, int, int, cudaStream_t);

}  // namespace mww
