// mww_serving_records.h -- the packed endpointer record of mww_export_endpointer_rows / mww_import_endpointer_rows (rule in
// include/mww.h, "moving endpointer rows") and the per-row bodies of the two kernels that fill and read it
// (mww_serving_records.cu).  One record holds one stream's row:
//
//     int32  member, armed, mute, 0                                 member of the stream set; armed (segmenter state follows);
//                                                                   the mute word of a positioned exporter, else 0
//     int32  elapsed, run, silence, heard                           zero unless armed
//     int64  seen; uint64 flags                                     the VAD count and the last 64 speech flags
//     int64  start_age, speech_end_age                              S' - start_sample, S' - speech_end_sample; zero unless armed
//     float32 hist[vad_window - 1]                                  oldest first (no bytes when vad_window = 1)
//
// every part padded to 16 bytes, S' the exporting endpointer's baseline samples_seen.  endpoint_record_layout() is the only
// place that knows the offsets.  A thread moves one record in 16-byte parts.  CUDA-free apart from MWW_HD and the two
// 16-byte accessors below, so that tests/emul_serving_records.cc runs the same functions on the CPU.
#pragma once

#include <stdint.h>

#include "mww_endpoint.h"

namespace mww {

inline long long endpoint_record_pad16(long long bytes) { return (bytes + 15) / 16 * 16; }

// byte offsets of the parts of a record and its size, for a rule of window vad_window
struct EpRecLayout {
    long long record_bytes;
    int head, seg, vad, ages, hist;
};
inline EpRecLayout endpoint_record_layout(int vad_window) {
    EpRecLayout L;
    long long off = 0;
    L.head = (int)off; off += endpoint_record_pad16(4 * sizeof(int32_t));
    L.seg = (int)off;  off += endpoint_record_pad16(4 * sizeof(int32_t));
    L.vad = (int)off;  off += endpoint_record_pad16(sizeof(long long) + sizeof(unsigned long long));
    L.ages = (int)off; off += endpoint_record_pad16(2 * sizeof(long long));
    L.hist = (int)off; off += endpoint_record_pad16((long long)(vad_window - 1) * (long long)sizeof(float));
    L.record_bytes = off;
    return L;
}

// what the kernels take: the endpointer's rule and state, its baseline and the layout
struct EpRecJob {
    EndpointArgs a;
    long long base = 0;            // S': samples_seen of the endpointer's last update or whole reset
    EpRecLayout L{};
};

// one 16-byte part of a record
struct EpRecPart { uint32_t w[4]; };
MWW_HD void endpoint_record_put(uint32_t *dst, const EpRecPart &p) {
#if defined(__CUDA_ARCH__)
    *reinterpret_cast<uint4 *>(dst) = make_uint4(p.w[0], p.w[1], p.w[2], p.w[3]);
#else
    for (int q = 0; q < 4; ++q) dst[q] = p.w[q];
#endif
}
MWW_HD EpRecPart endpoint_record_get(const uint32_t *src) {
#if defined(__CUDA_ARCH__)
    const uint4 v = *reinterpret_cast<const uint4 *>(src);
    return EpRecPart{{v.x, v.y, v.z, v.w}};
#else
    return EpRecPart{{src[0], src[1], src[2], src[3]}};
#endif
}
MWW_HD uint32_t endpoint_lo(long long v) { return (uint32_t)((unsigned long long)v & 0xFFFFFFFFull); }
MWW_HD uint32_t endpoint_hi(long long v) { return (uint32_t)((unsigned long long)v >> 32); }
MWW_HD long long endpoint_join(uint32_t lo, uint32_t hi) { return (long long)(((unsigned long long)hi << 32) | lo); }

// endpointer -> the record of global id `id` (in range).  A non-member gets a zero record; an unarmed row zero segmenter
// state.  kAt: an armed row's mute word goes into the head's third word.  Reads only.
template <bool kAt>
MWW_HD void endpoint_record_pack_t(const EpRecJob &J, const int32_t *mute, int id, uint32_t *rec) {
    const EndpointArgs &a = J.a;
    const int r = endpoint_row(a, id);
    const bool member = r >= 0, armed = member && a.armed[r] >= 0;
    uint32_t m = 0u;
    if constexpr (kAt) m = armed ? (uint32_t)mute[r] : 0u;
    endpoint_record_put(rec + J.L.head / 4, EpRecPart{{member ? 1u : 0u, armed ? 1u : 0u, m, 0u}});
    EpRecPart seg{{0u, 0u, 0u, 0u}}, ages{{0u, 0u, 0u, 0u}}, vad{{0u, 0u, 0u, 0u}};
    if (armed) {
        seg = EpRecPart{{(uint32_t)a.elapsed[r], (uint32_t)a.run[r], (uint32_t)a.silence[r], (uint32_t)a.heard[r]}};
        const long long s = J.base - a.start[r], e = J.base - a.speech_end[r];
        ages = EpRecPart{{endpoint_lo(s), endpoint_hi(s), endpoint_lo(e), endpoint_hi(e)}};
    }
    if (member) {
        const long long seen = a.seen[r], flags = (long long)a.flags[r];
        vad = EpRecPart{{endpoint_lo(seen), endpoint_hi(seen), endpoint_lo(flags), endpoint_hi(flags)}};
    }
    endpoint_record_put(rec + J.L.seg / 4, seg);
    endpoint_record_put(rec + J.L.vad / 4, vad);
    endpoint_record_put(rec + J.L.ages / 4, ages);
    const int hl = a.rule.vad_window - 1;
    const uint32_t *hist = reinterpret_cast<const uint32_t *>(a.hist);
    for (int c = 0; 4 * c < hl; ++c) {
        EpRecPart p;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int j = 4 * c + q;
            p.w[q] = member && j < hl ? hist[(long long)j * a.n_rows + r] : 0u;
        }
        endpoint_record_put(rec + J.L.hist / 4 + 4 * c, p);
    }
}
MWW_HD void endpoint_record_pack(const EpRecJob &J, int id, uint32_t *rec) { endpoint_record_pack_t<false>(J, nullptr, id, rec); }

// record -> endpointer, global id `id` (in range).  A non-member ignores the record; a member whose record has member = 0
// gets what reset(ids) gives; a member whose record has member = 1 takes the VAD state, and, when the record is armed, the
// segmenter with armed = id and positions S' - age.  arm_tag is not written.  kAt: the row's mute word is the head's third
// word when the record is armed (0 in a plain exporter's records) and 0 otherwise.
template <bool kAt>
MWW_HD void endpoint_record_unpack_t(const EpRecJob &J, int32_t *mute, int id, const uint32_t *rec) {
    const EndpointArgs &a = J.a;
    const int r = endpoint_row(a, id);
    if (r < 0) return;
    const EpRecPart head = endpoint_record_get(rec + J.L.head / 4);
    if (!head.w[0]) {
        endpoint_clear_row_t<kAt>(a, mute, r, 1);
        return;
    }
    const EpRecPart vad = endpoint_record_get(rec + J.L.vad / 4);
    a.seen[r] = endpoint_join(vad.w[0], vad.w[1]);
    a.flags[r] = (unsigned long long)endpoint_join(vad.w[2], vad.w[3]);
    const int hl = a.rule.vad_window - 1;
    uint32_t *hist = reinterpret_cast<uint32_t *>(a.hist);
    for (int c = 0; 4 * c < hl; ++c) {
        const EpRecPart p = endpoint_record_get(rec + J.L.hist / 4 + 4 * c);
#pragma unroll
        for (int q = 0; q < 4; ++q)
            if (4 * c + q < hl) hist[(long long)(4 * c + q) * a.n_rows + r] = p.w[q];
    }
    if (!head.w[1]) {
        a.armed[r] = -1;
        endpoint_store_seg(a, r, endpoint_fresh_seg());
        if constexpr (kAt) mute[r] = 0;
        return;
    }
    const EpRecPart seg = endpoint_record_get(rec + J.L.seg / 4);
    const EpRecPart ages = endpoint_record_get(rec + J.L.ages / 4);
    a.armed[r] = id;
    endpoint_store_seg(a, r, EndpointSeg{(int)seg.w[0], (int)seg.w[1], (int)seg.w[2], (int)seg.w[3],
                                         J.base - endpoint_join(ages.w[0], ages.w[1]), J.base - endpoint_join(ages.w[2], ages.w[3])});
    if constexpr (kAt) mute[r] = (int32_t)head.w[2];
}
MWW_HD void endpoint_record_unpack(const EpRecJob &J, int id, const uint32_t *rec) { endpoint_record_unpack_t<false>(J, nullptr, id, rec); }

// The first field in which the layout the records were exported with differs from the importing endpointer's own, nullptr
// when the records fit.  The baselines (samples_seen, steps) are for information and not compared.
inline const char *endpoint_layout_mismatch(const mww_endpointer_layout &src, const mww_endpointer_layout &dst) {
    if (src.vad_window != dst.vad_window) return "vad_window";
    if (src.stride != dst.stride) return "stride";
    if (src.hop_samples != dst.hop_samples) return "hop_samples";
    if (src.buffered != dst.buffered) return "buffered";
    if (src.pending != dst.pending) return "pending";
    if (src.record_bytes != dst.record_bytes) return "record_bytes";
    return nullptr;
}

}  // namespace mww
