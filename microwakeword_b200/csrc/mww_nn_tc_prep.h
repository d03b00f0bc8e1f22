// mww_nn_tc_prep.h -- the wgmma clip kernel's operand layout, shared by the kernel (mww_nn_tc.cu: the CUDA cores write the A
// operand with it, mww_create lays the weights out with it) and by the host-side test that reads the operands back the way the tensor
// core does (tests/host_emul).  No CUDA dependency.
#pragma once

#include <stddef.h>
#include <stdint.h>
#include <string.h>

#include <vector>

#include "mww_common.h"

namespace mww {

// 128-byte-swizzled K-major slot (wgmma shared-memory matrix descriptor with SWIZZLE_128B, stride byte offset 1024): rows of 128
// bytes = 32 fp32 along K; within each group of 8 rows the 16-byte chunk index is XORed with (row & 7).  Byte offset of element
// (row, kk), kk in [0, 32).
MWW_HD uint32_t sw128_off(int row, int kk) {
    return (uint32_t)row * 128u + (uint32_t)((((kk >> 2) ^ (row & 7)) << 4) + ((kk & 3) << 2));
}

// [K][N] fp32 weights -> K cut into slots of 32; per slot a hi plane [N rows][128 B swizzled] followed by the lo plane, where
// hi = the value with its low 13 mantissa bits cleared (a TF32 the tensor core reads exactly) and lo = value - hi (exact in fp32);
// positions k >= K of the last slot are zero.
inline void tc_layout(const float *w, int K, int N, std::vector<unsigned char> *out) {
    const int slots = (K + 31) / 32, plane = N * 128;
    out->assign((size_t)slots * 2 * plane, 0);
    for (int k = 0; k < K; ++k)
        for (int n = 0; n < N; ++n) {
            const float v = w[(size_t)k * N + n];
            uint32_t u;
            memcpy(&u, &v, 4);
            const uint32_t hu = u & 0xFFFFE000u;
            float hi, lo;
            memcpy(&hi, &hu, 4);
            lo = v - hi;
            unsigned char *slot = out->data() + (size_t)(k >> 5) * 2 * plane;
            memcpy(slot + sw128_off(n, k & 31), &hi, 4);
            memcpy(slot + plane + sw128_off(n, k & 31), &lo, 4);
        }
}

}  // namespace mww
