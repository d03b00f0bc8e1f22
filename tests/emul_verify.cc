// tests/emul_verify.cc -- TEST INFRASTRUCTURE: the per-element bodies of the two verification kernels
// (microwakeword_b200/csrc/mww_verify.h) run on the CPU, an index at a time as the kernels' threads run them, for
// tests/test_verify.py.  Never used by the product.
#include "../microwakeword_b200/csrc/mww_verify.h"

using namespace mww;

// ids [capacity] of a detector's event slots, `count` events having fired
extern "C" void emul_verify_slots(long long count, const mww_event *events, int capacity, int model, int32_t *ids) {
    for (int i = 0; i < capacity; ++i) ids[i] = verify_slot_id(i, count, capacity, events, model);
}

// out_scores / out_confirmed [n] from ids [n] and scores [n]
extern "C" void emul_verify_confirm(const int32_t *ids, int n, int n_streams, const float *scores, double cutoff, float *out_scores,
                                    int32_t *out_confirmed) {
    for (int i = 0; i < n; ++i) {
        const VerifyOut o = verify_confirm(ids[i], n_streams, scores[i], cutoff);
        out_scores[i] = o.score;
        out_confirmed[i] = o.confirmed;
    }
}
