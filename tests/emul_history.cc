// tests/emul_history.cc -- TEST INFRASTRUCTURE: the ring index math of microwakeword_b200/csrc/mww_history.h and the per-unit
// bodies of the append and read kernels (mww_history.cu) run on the CPU, unit by unit as the kernels' threads run them, for
// tests/test_audio_history.py.  Never used by the product.
#include <stdint.h>

#include "../microwakeword_b200/csrc/mww_history.h"

using namespace mww;

namespace {
// the append kernel over every stream: 8-sample units (the vector form, as load8 + one 16-byte store) or single samples
template <typename T>
int append(int16_t *ring, int n_streams, int C, long long seen, const T *audio, long long stride, int n16, int allow_vec) {
    if (n16 <= 0) return 0;
    const HistoryAppend p = history_append_plan(seen, n16, C);
    const int vec = allow_vec && history_append_vec_shape(p, stride);
    const int units = vec ? p.m / 8 : p.m;
    for (long long s = 0; s < n_streams; ++s)
        for (int u = 0; u < units; ++u) {
            int16_t *row = ring + s * C;
            const T *src = audio + s * stride;
            if (vec) {
                int16_t *dst = row + history_slot(p.slot0, 8 * u, C);
                for (int q = 0; q < 8; ++q) dst[q] = pcm16(src[p.src0 + 8 * u + q]);
            } else {
                history_append_one(row, src, p, u, C);
            }
        }
    return vec;
}
}  // namespace

extern "C" int emul_history_capacity_ok(long long C) { return history_capacity_ok(C); }

// type: 0 int16, 1 float32, 2 mu-law, 3 A-law.  Returns 1 when the vector form ran.
extern "C" int emul_history_append(int type, int16_t *ring, int n_streams, int C, long long seen, const void *audio, long long stride, int n16,
                                   int allow_vec) {
    switch (type) {
    case 0: return append(ring, n_streams, C, seen, static_cast<const int16_t *>(audio), stride, n16, allow_vec);
    case 1: return append(ring, n_streams, C, seen, static_cast<const float *>(audio), stride, n16, allow_vec);
    case 2: return append(ring, n_streams, C, seen, static_cast<const Ulaw8 *>(audio), stride, n16, allow_vec);
    default: return append(ring, n_streams, C, seen, static_cast<const Alaw8 *>(audio), stride, n16, allow_vec);
    }
}

// the read kernel: row i of out = the last n_samples of ring row ids[i] (zeros for an id outside [0, n_streams)), in the
// vector form (8 entries from the unit's first slot) when its shape holds.  Returns 1 when it did.
extern "C" int emul_history_read(const int16_t *ring, int C, int n_streams, long long seen, const int32_t *ids, int n, int n_samples,
                                 int16_t *out, long long out_stride) {
    if (n_samples <= 0) return 0;
    const int slot0 = history_read_slot0(seen, n_samples, C);
    const int vec = history_read_vec_shape(slot0, n_samples, out_stride);
    for (long long r = 0; r < n; ++r) {
        if (vec) {          // one 16-byte load from the unit's first slot, as the kernel
            for (int u = 0; u < n_samples / 8; ++u) {
                const int base = history_slot(slot0, 8 * u, C);
                for (int q = 0; q < 8; ++q)
                    out[r * out_stride + 8 * u + q] = ids[r] >= 0 && ids[r] < n_streams ? ring[(long long)ids[r] * C + base + q] : 0;
            }
        } else {
            for (int k = 0; k < n_samples; ++k) out[r * out_stride + k] = history_read_one(ring, C, ids[r], n_streams, slot0, k);
        }
    }
    return vec;
}
