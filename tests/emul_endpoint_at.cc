// tests/emul_endpoint_at.cc -- TEST INFRASTRUCTURE: the positioned forms of the endpointer's per-row bodies
// (microwakeword_b200/csrc/mww_endpoint.h and mww_serving_records.h with kAt = true) run on the CPU, a row or an id at a time
// as the kernels' threads run them, for tests/test_endpoint_at.py.  It includes tests/emul_endpoint.cc, so one library holds
// the plain forms too.  Never used by the product.
#include "emul_endpoint.cc"

#include "../microwakeword_b200/csrc/mww_serving_records.h"

extern "C" void emul_at_update(const int *cfg, double cutoff, long long step_samples, void **p, int32_t *mute, const float *probs,
                               long long pitch, int n, long long pos0) {
    const EndpointArgs a = args(cfg, cutoff, step_samples, p);
    for (int r = 0; r < a.n_rows; ++r) endpoint_update_row_t<true>(a, mute, r, probs, pitch, n, pos0);
}

extern "C" void emul_at_arm(const int *cfg, double cutoff, long long step_samples, void **p, int32_t *mute, const int32_t *ids, int n, int steps,
                            int tag, const long long *pos) {
    const EndpointArgs a = args(cfg, cutoff, step_samples, p);
    EndpointReplay R;
    R.steps = steps; R.tag = tag;
    for (int i = 0; i < kEndpointMaxLookback; ++i) R.pos[i] = pos[i];
    for (int i = 0; i < n; ++i) endpoint_arm_one_t<true>(a, mute, R, ids[i]);
}

extern "C" void emul_at_clear(const int *cfg, double cutoff, long long step_samples, void **p, int32_t *mute, const int32_t *ids, int n,
                              int reset) {
    const EndpointArgs a = args(cfg, cutoff, step_samples, p);
    for (int i = 0; i < n; ++i) {
        const int r = ids ? endpoint_row(a, ids[i]) : i;
        if (r >= 0) endpoint_clear_row_t<true>(a, mute, r, reset);
    }
}

// arm_at's two passes over the n listed (id, position) slots; the second pass visits the slots in `order` (a permutation),
// standing for any order the kernel's threads may take
extern "C" void emul_at_arm_at(const int *cfg, double cutoff, long long step_samples, void **p, int32_t *mute, unsigned long long *key,
                               const int32_t *ids, const long long *positions, int n, const int *order, int steps, int tag, const long long *pos,
                               long long q, long long skip) {
    const EndpointArgs a = args(cfg, cutoff, step_samples, p);
    EndpointAt A;
    A.R.steps = steps; A.R.tag = tag;
    for (int i = 0; i < kEndpointMaxLookback; ++i) A.R.pos[i] = pos[i];
    A.q = q; A.skip = skip; A.mute = mute; A.key = key;
    for (int i = 0; i < n; ++i) endpoint_at_reduce_one(a, A, ids[i], positions[i]);
    for (int i = 0; i < n; ++i) endpoint_arm_at_one(a, A, ids[order[i]], positions[order[i]]);
}

// records [n][record_bytes] of the listed ids, plain (at = 0) or positioned (at = 1)
extern "C" long long emul_at_record_bytes(int vad_window) { return endpoint_record_layout(vad_window).record_bytes; }

extern "C" void emul_at_pack(const int *cfg, double cutoff, long long step_samples, void **p, const int32_t *mute, long long base, const int32_t *ids,
                             int n, uint32_t *rec, int at) {
    EpRecJob J;
    J.a = args(cfg, cutoff, step_samples, p);
    J.base = base;
    J.L = endpoint_record_layout(cfg[0]);
    for (int i = 0; i < n; ++i) {
        uint32_t *dst = rec + (long long)i * (J.L.record_bytes / 4);
        if (at) endpoint_record_pack_t<true>(J, mute, ids[i], dst);
        else endpoint_record_pack(J, ids[i], dst);
    }
}

extern "C" void emul_at_unpack(const int *cfg, double cutoff, long long step_samples, void **p, int32_t *mute, long long base, const int32_t *ids,
                               int n, const uint32_t *rec, int at) {
    EpRecJob J;
    J.a = args(cfg, cutoff, step_samples, p);
    J.base = base;
    J.L = endpoint_record_layout(cfg[0]);
    for (int i = 0; i < n; ++i) {
        const uint32_t *src = rec + (long long)i * (J.L.record_bytes / 4);
        if (at) endpoint_record_unpack_t<true>(J, mute, ids[i], src);
        else endpoint_record_unpack(J, ids[i], src);
    }
}
