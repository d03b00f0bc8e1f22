// tests/emul_detector_records.cc -- TEST INFRASTRUCTURE: the record layout of microwakeword_b200/csrc/mww_detector_records.h
// and the per-word bodies of the pack and unpack kernels (mww_detector_records.cu) run on the CPU, word by word as the
// kernels' threads run them, for tests/test_detector_records.py.  Never used by the product.
#include <string.h>

#include <vector>

#include "../microwakeword_b200/csrc/mww_detector_records.h"

using namespace mww;

namespace {
// the descriptors of a detector whose model k has role[k], window[k], cooldown[k] and n_rows[k] rows of host state
std::vector<DetectModel> models(int K, const int *role, const int *window, const int *cooldown, const int *n_rows,
                                const int32_t *const *inv, float *const *hist, long long *const *seen, int32_t *const *flag) {
    std::vector<DetectModel> m((size_t)K);
    for (int k = 0; k < K; ++k) {
        DetectModel &s = m[(size_t)k];
        s.role = role[k]; s.rule.window = window[k]; s.rule.cooldown_slices = cooldown[k];
        if (n_rows) { s.n_rows = n_rows[k]; s.inv = inv[k]; s.hist = hist[k]; s.seen = seen[k]; s.flag = flag[k]; }
    }
    return m;
}
}  // namespace

// out: record_bytes, then hist_off[K], then tail_off[K] (-1 for an OFF model)
extern "C" void emul_detrec_layout(const int *role, const int *window, int K, long long *out) {
    const std::vector<DetectModel> m = models(K, role, window, window, nullptr, nullptr, nullptr, nullptr, nullptr);
    const DetRecLayout L = detector_record_layout(m.data(), K);
    out[0] = L.record_bytes;
    for (int k = 0; k < K; ++k) { out[1 + k] = L.hist_off[k]; out[1 + K + k] = L.tail_off[k]; }
}

// records [n][record_bytes / 4] of ids[0, n); returns the words per record
extern "C" int emul_detrec_pack(int K, const int *role, const int *window, const int *cooldown, const int *n_rows, const int32_t *const *inv,
                                float *const *hist, long long *const *seen, int32_t *const *flag, const int32_t *ids, int n, uint32_t *rec) {
    const std::vector<DetectModel> m = models(K, role, window, cooldown, n_rows, inv, hist, seen, flag);
    const DetRecJob J = detector_record_job(m.data(), K);
    for (int j = 0; j < n; ++j)
        for (int w = 0; w < J.words; ++w) detector_record_pack_word(J, w, ids[j], rec + (long long)j * J.words);
    return J.words;
}

extern "C" int emul_detrec_unpack(int K, const int *role, const int *window, const int *cooldown, const int *n_rows, const int32_t *const *inv,
                                  float *const *hist, long long *const *seen, int32_t *const *flag, const int32_t *ids, int n, const uint32_t *rec) {
    const std::vector<DetectModel> m = models(K, role, window, cooldown, n_rows, inv, hist, seen, flag);
    const DetRecJob J = detector_record_job(m.data(), K);
    for (int j = 0; j < n; ++j)
        for (int w = 0; w < J.words; ++w) detector_record_unpack_word(J, w, ids[j], rec + (long long)j * J.words);
    return J.words;
}

// 0 when the records fit, else 1 with the field's name in `field` and the model in *index (-1: not a per-model field)
extern "C" int emul_detrec_mismatch(const mww_detector_layout *src, const mww_detector_layout *dst, int *index, char *field, int cap) {
    const char *f = detector_layout_mismatch(*src, *dst, index);
    if (!f) return 0;
    strncpy(field, f, (size_t)cap - 1);
    field[cap - 1] = 0;
    return 1;
}
