// mww_streams.h -- index math of per-model stream sets (mww_create_multi_streams): which members of a model a stream tile
// holds, where the row-gather and state-remap kernels (mww_streams.cu) read and write, and the compact index of a global
// stream id.  A model's members are a strictly increasing list of global stream ids; its ring state, pending rows and
// probabilities are indexed by position in that list (the compact index).  CUDA-free apart from MWW_HD, so that
// tests/emul_streams.cc runs the same functions on the CPU.
#pragma once

#include "mww_common.h"

namespace mww {

// first j in [0, n) with ids[j] >= v, n if none (ids strictly increasing)
MWW_HD int lower_bound_ids(const int32_t *ids, int n, int v) {
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (ids[mid] < v) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// The members of a model (sorted ids[0, n)) inside the stream tile [first, first + tile) are its compact indices [*a, *b).
// Returns true when they are also consecutive stream ids, so the tile's feature rows can be read in place (no members
// counts as consecutive); false when they have to be gathered.
inline bool tile_members(const int32_t *ids, int n, int first, int tile, int *a, int *b) {
    *a = lower_bound_ids(ids, n, first);
    *b = lower_bound_ids(ids, n, first + tile);
    return *b == *a || ids[*b - 1] - ids[*a] == *b - *a - 1;
}

// ids[0, n) is a valid stream set of a handle of n_streams streams: strictly increasing, inside [0, n_streams)
inline bool valid_stream_set(const int32_t *ids, int n, int n_streams) {
    for (int i = 0; i < n; ++i)
        if (ids[i] < 0 || ids[i] >= n_streams || (i > 0 && ids[i] <= ids[i - 1])) return false;
    return true;
}

// Row gather of one tile: 16-byte chunk i of the compact buffer [m][chunks_per_stream] comes from chunk *src of the tile's
// feature rows, which start at stream `first` with chunks_per_stream chunks per stream; ids + a are the tile's members.
MWW_HD long long gather_source(long long i, long long chunks_per_stream, const int32_t *ids, int a, int first) {
    const long long j = i / chunks_per_stream;
    return (long long)(ids[a + j] - first) * chunks_per_stream + (i - j * chunks_per_stream);
}

// State remap of a membership change: word i of the new rows [n_new][words_per_row] comes from this word of the old rows,
// or -1 for a stream that joins (old_index[j]: old compact index of new member j, -1 if it was not a member)
MWW_HD long long remap_source(long long i, long long words_per_row, const int32_t *old_index) {
    const long long j = i / words_per_row;
    const int32_t o = old_index[j];
    return o < 0 ? -1 : (long long)o * words_per_row + (i - j * words_per_row);
}

// compact index of global stream id `id` from a model's inverse map inv[n_streams]; -1 for a non-member or an id out of range
MWW_HD int32_t compact_id(int32_t id, const int32_t *inv, int n_streams) { return id >= 0 && id < n_streams ? inv[id] : -1; }

}  // namespace mww
