// tests/emul_streams.cc -- TEST INFRASTRUCTURE: the index math of per-model stream sets (microwakeword_b200/csrc/mww_streams.h)
// run on the CPU, for tests/test_model_streams.py.
#include "../microwakeword_b200/csrc/mww_streams.h"

using namespace mww;

// tile planner: for each tile [first, first + tile) of n_streams streams, a[t], b[t] and consecutive[t]
extern "C" int emul_tile_plan(const int32_t *ids, int n, int n_streams, int tile, int32_t *a, int32_t *b, int32_t *consecutive) {
    int t = 0;
    for (int first = 0; first < n_streams; first += tile, ++t) {
        const int len = n_streams - first < tile ? n_streams - first : tile;
        int ta, tb;
        consecutive[t] = tile_members(ids, n, first, len, &ta, &tb);
        a[t] = ta; b[t] = tb;
    }
    return t;
}

extern "C" int emul_valid_stream_set(const int32_t *ids, int n, int n_streams) { return valid_stream_set(ids, n, n_streams); }

// the row gather of one tile, thread by thread: out[i] = feat[gather_source(i)], 16-byte chunks as pairs of uint64
extern "C" void emul_gather(const uint64_t *feat, const int32_t *ids, int a, int first, int m, long long chunks_per_stream, uint64_t *out) {
    for (long long i = 0; i < (long long)m * chunks_per_stream; ++i) {
        const long long s = gather_source(i, chunks_per_stream, ids, a, first);
        out[2 * i] = feat[2 * s];
        out[2 * i + 1] = feat[2 * s + 1];
    }
}

// the state remap, word by word: dst rows of joiners (old_index -1) are left as they are
extern "C" void emul_remap(uint32_t *dst, const uint32_t *src, long long words_per_row, const int32_t *old_index, int n_new) {
    for (long long i = 0; i < words_per_row * n_new; ++i) {
        const long long s = remap_source(i, words_per_row, old_index);
        if (s >= 0) dst[i] = src[s];
    }
}

extern "C" void emul_compact_ids(int32_t *out, const int32_t *ids, int n, const int32_t *inv, int n_streams) {
    for (int i = 0; i < n; ++i) out[i] = compact_id(ids[i], inv, n_streams);
}
