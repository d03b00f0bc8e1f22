// Device harness for tests/test_gpu_device_forms.py: evaluates the product's __device__ forms of the frontend's scalar
// helpers (the #if __CUDA_ARCH__ branches of mww_common.h and mww_frontend_dev.cuh, compiled for sm_90a exactly as the
// kernels include them) against the portable references of scalar_refs.h over whole input domains.  Every kernel walks
// indices [0, n) with a grid stride, forms its input from the index (or reads it from a caller list of n_list entries, index
// checked), counts mismatches and keeps the smallest mismatching index (atomicMin).
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -shared -Xcompiler -fPIC -o libdevice_forms.so \
//        device_forms.cu ../../microwakeword_b200/csrc/mww_tables.cc
#include <cuda_runtime.h>

#include "../../microwakeword_b200/csrc/mww_frontend_dev.cuh"
#include "scalar_refs.h"

namespace {

struct Verdict { unsigned long long count, first; };

int16_t *g_gain = nullptr;
uint16_t *g_log = nullptr;
Verdict *g_verdict = nullptr;

__device__ __forceinline__ void miss(Verdict *v, unsigned long long i) {
    atomicAdd(&v->count, 1ull);
    atomicMin(&v->first, i);
}

__device__ __forceinline__ uint64_t splitmix64(uint64_t z) {
    z += 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

#define GRID_STRIDE(i, n) for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < (n); \
                               i += (unsigned long long)gridDim.x * blockDim.x)

// x = lo + i: wide_dynamic_function and pcan_shrink
__global__ void k_wdf_pcan(unsigned long long lo, unsigned long long n, const int16_t *gain, Verdict *v) {
    GRID_STRIDE(i, n) {
        const uint32_t x = (uint32_t)(lo + i);
        if (mww::wide_dynamic_function(x, gain) != ref::wide_dynamic_function(x, gain) || mww::pcan_shrink(x) != ref::pcan_shrink(x))
            miss(v, i);
    }
}

// x = lo + i, x >= 2
__global__ void k_log_scale(unsigned long long lo, unsigned long long n, const uint16_t *lut, Verdict *v) {
    GRID_STRIDE(i, n) {
        const uint32_t x = (uint32_t)(lo + i);
        if (mww::log_scale(x, lut) != ref::log_scale(x, lut)) miss(v, i);
    }
}

// i = e * 65536 + value: every v < 2^16 against every listed estimate
__global__ void k_k2_output(const uint32_t *est, long long n_est, const int16_t *gain, const uint16_t *lut, Verdict *v) {
    const unsigned long long n = (unsigned long long)n_est << 16;
    GRID_STRIDE(i, n) {
        const unsigned long long e = i >> 16;
        const uint32_t val = (uint32_t)(i & 0xFFFFu);
        if (mww::k2_output(val, est[e], gain, lut) != ref::k2_output(val, est[e], gain, lut)) miss(v, i);
    }
}

// x = lo + i (lo + n <= 2^48)
__global__ void k_isqrt_range(unsigned long long lo, unsigned long long n, Verdict *v) {
    GRID_STRIDE(i, n) {
        const uint64_t x = lo + i;
        if (!ref::isqrt_below48_ok(x, mww::isqrt64_round_below48(x))) miss(v, i);
    }
}

// i = 6 * (m - 1) + k for 1 <= m < 2^24: n^2 - n, n^2 - n + 1, n^2 - 1, n^2, n^2 + n, n^2 + n + 1 with n = m, the inputs
// next to a half-integer or an integer root
__global__ void k_isqrt_near_roots(unsigned long long n, Verdict *v) {
    GRID_STRIDE(i, n) {
        const uint64_t m = i / 6 + 1, k = i % 6, sq = m * m;
        const uint64_t x = k == 0 ? sq - m : k == 1 ? sq - m + 1 : k == 2 ? sq - 1 : k == 3 ? sq : k == 4 ? sq + m : sq + m + 1;
        if (x >= (1ull << 48)) continue;
        if (!ref::isqrt_below48_ok(x, mww::isqrt64_round_below48(x))) miss(v, i);
    }
}

// every float32 bit pattern lo + i
__global__ void k_pcm16(unsigned long long lo, unsigned long long n, Verdict *v) {
    GRID_STRIDE(i, n) {
        const float x = __uint_as_float((uint32_t)(lo + i));
        if (mww::pcm16_from_f32(x) != ref::pcm16_from_f32(x)) miss(v, i);
    }
}

// windowing: mulhi_s32 of the sample in the high half (as k1_window_fft1 forms it from the low and from the high sample of a
// packed word whose other half is not zero) times w << 4, against (s * w) >> 12; i = (s + 32768) * 4097 + w
__global__ void k_window(Verdict *v) {
    const unsigned long long n = 65536ull * 4097ull;
    GRID_STRIDE(i, n) {
        const int32_t s = (int32_t)(i / 4097) - 32768, w = (int32_t)(i % 4097);
        const uint32_t lo_word = 0x5A5A0000u | ((uint32_t)s & 0xFFFFu), hi_word = ((uint32_t)s << 16) | 0xA5A5u;
        const int32_t want = (s * w) >> 12;
        if (mww::mulhi_s32((int32_t)(lo_word << 16), w << 4) != want || mww::mulhi_s32((int32_t)(hi_word & 0xFFFF0000u), w << 4) != want)
            miss(v, i);
    }
}

// clz32, msb32, shl_clamp32 (every s in 0..33), mulhi_s32 and vmax_u16x2 on the listed values (i < n_list) and on random
// words (i >= n_list); the second operand is the next list entry or another random word
__global__ void k_bits(const uint32_t *list, long long n_list, unsigned long long n, Verdict *v) {
    GRID_STRIDE(i, n) {
        const bool listed = i < (unsigned long long)n_list;
        const uint64_t h = splitmix64(i);
        const uint32_t x = listed ? list[i] : (uint32_t)h;
        const uint32_t y = listed ? list[(i + 1) % (unsigned long long)n_list] : (uint32_t)(h >> 32);
        bool bad = mww::clz32(x) != ref::clz(x) || mww::msb32(x) != ref::msb(x) ||
                   mww::vmax_u16x2(x, y) != ref::vmax_u16x2(x, y) || mww::vmax_u16x2(y, x) != ref::vmax_u16x2(y, x) ||
                   mww::mulhi_s32((int32_t)x, (int32_t)y) != ref::mulhi((int32_t)x, (int32_t)y);
        for (int s = 0; s <= 33; ++s) bad |= mww::shl_clamp32(x, s) != ref::shl_clamp(x, s);
        if (bad) miss(v, i);
    }
}

// device outputs on a caller list, for the comparison with the oracle library on the host.  fn: 0 wide_dynamic_function
// (as int32 bits), 1 pcan_shrink, 2 log_scale, 3 isqrt64_round_below48; 4 the double reference of pcm16_from_f32 (input:
// float bits; output: the int16 sign-extended)
__global__ void k_eval(int fn, const uint64_t *in, uint32_t *out, long long n, const int16_t *gain, const uint16_t *lut) {
    GRID_STRIDE(i, (unsigned long long)n) {
        const uint64_t x = in[i];
        uint32_t r = 0;
        if (fn == 0) r = (uint32_t)mww::wide_dynamic_function((uint32_t)x, gain);
        else if (fn == 1) r = mww::pcan_shrink((uint32_t)x);
        else if (fn == 2) r = mww::log_scale((uint32_t)x, lut);
        else if (fn == 3) r = mww::isqrt64_round_below48(x);
        else r = (uint32_t)(int32_t)ref::pcm16_from_f32(__uint_as_float((uint32_t)x));
        out[i] = r;
    }
}

unsigned grid_blocks() {
    int dev = 0, sms = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    return (unsigned)(sms > 0 ? sms * 16 : 1024);
}

}  // namespace

extern "C" {

// builds the product's tables and uploads the PCAN and log LUTs; 0 or a cudaError_t
int forms_init() {
    if (g_verdict) return 0;
    mww::HostTables t;
    mww::build_host_tables(&t);
    if (!t.ok) return -1;
    cudaError_t e;
    if ((e = cudaMalloc(&g_gain, sizeof t.gain_lut)) || (e = cudaMalloc(&g_log, sizeof t.log_lut)) || (e = cudaMalloc(&g_verdict, sizeof(Verdict))))
        return (int)e;
    if ((e = cudaMemcpy(g_gain, t.gain_lut, sizeof t.gain_lut, cudaMemcpyHostToDevice)) ||
        (e = cudaMemcpy(g_log, t.log_lut, sizeof t.log_lut, cudaMemcpyHostToDevice)))
        return (int)e;
    return 0;
}

// one domain sweep.  which: 0 wdf+pcan (lo, n), 1 log_scale (lo, n), 2 k2_output (list of estimates), 3 isqrt range (lo, n),
// 4 isqrt near roots (n), 5 pcm16 (lo, n), 6 windowing, 7 bit helpers (list, n).  Writes the mismatch count and the first
// mismatching index (~0 if none); returns 0 or a cudaError_t.
int forms_check(int which, unsigned long long lo, unsigned long long n, const void *list, long long n_list,
                unsigned long long *count, unsigned long long *first) {
    if (!g_verdict) return -1;
    const Verdict init{0ull, ~0ull};
    cudaError_t e = cudaMemcpy(g_verdict, &init, sizeof init, cudaMemcpyHostToDevice);
    if (e) return (int)e;
    const unsigned grid = grid_blocks();
    switch (which) {
        case 0: k_wdf_pcan<<<grid, 256>>>(lo, n, g_gain, g_verdict); break;
        case 1: k_log_scale<<<grid, 256>>>(lo, n, g_log, g_verdict); break;
        case 2: k_k2_output<<<grid, 256>>>(static_cast<const uint32_t *>(list), n_list, g_gain, g_log, g_verdict); break;
        case 3: k_isqrt_range<<<grid, 256>>>(lo, n, g_verdict); break;
        case 4: k_isqrt_near_roots<<<grid, 256>>>(n, g_verdict); break;
        case 5: k_pcm16<<<grid, 256>>>(lo, n, g_verdict); break;
        case 6: k_window<<<grid, 256>>>(g_verdict); break;
        case 7: k_bits<<<grid, 256>>>(static_cast<const uint32_t *>(list), n_list, n, g_verdict); break;
        default: return -1;
    }
    if ((e = cudaGetLastError()) || (e = cudaDeviceSynchronize())) return (int)e;
    Verdict out;
    if ((e = cudaMemcpy(&out, g_verdict, sizeof out, cudaMemcpyDeviceToHost))) return (int)e;
    *count = out.count;
    *first = out.first;
    return 0;
}

// device pointers in (uint64 [n]) and out (uint32 [n])
int forms_eval(int fn, const void *in, void *out, long long n) {
    if (!g_verdict || fn < 0 || fn > 4) return -1;
    k_eval<<<grid_blocks(), 256>>>(fn, static_cast<const uint64_t *>(in), static_cast<uint32_t *>(out), n, g_gain, g_log);
    cudaError_t e = cudaGetLastError();
    if (!e) e = cudaDeviceSynchronize();
    return (int)e;
}

}  // extern "C"
