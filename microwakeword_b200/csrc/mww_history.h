// mww_history.h -- the audio history of a handle (mww_set_audio_history, rule in include/mww.h): a ring of the last C 16 kHz
// int16 samples of every stream, and the index math of the two kernels that fill and read it (mww_history.cu) and of the
// kernel that writes whole rows (mww_write_audio_history, mww_serving_records.cu).
//
// All streams advance in lockstep, so one counter, `seen` (16 kHz samples appended since the history was enabled), places
// every stream's ring: sample t of the run since enabling lives in slot t mod C of its stream's row.  A zeroed row reads as
// the endless run of zeros the rule starts with, whatever `seen` is.  C is a multiple of 8, so an 8-sample vector that starts
// on a slot that is a multiple of 8 never straddles the wrap.
//
// CUDA-free apart from MWW_HD, so that tests/emul_history.cc runs the same functions on the CPU.
#pragma once

#include "mww_frontend_dev.cuh"     // pcm16() of every sample type

namespace mww {

constexpr int kHistoryMaxCapacity = 1 << 22;

// 0 (off) or a multiple of 8 in [8, 2^22]
MWW_HD bool history_capacity_ok(long long C) { return C == 0 || (C >= 8 && C <= kHistoryMaxCapacity && C % 8 == 0); }

// x mod C in [0, C), for any sign of x
MWW_HD int history_mod(long long x, int C) {
    const long long r = x % C;
    return (int)(r < 0 ? r + C : r);
}

// slot of entry k of a run that starts in slot0 (0 <= slot0 < C, 0 <= k < C): the run wraps to slot 0 at most once
MWW_HD int history_slot(int slot0, int k, int C) {
    const int s = slot0 + k;
    return s >= C ? s - C : s;
}

// A call of n16 samples per stream, appended when `seen` samples came before it: only its last m = min(n16, C) samples can
// be read back, so only they are written, sample src0 + j of the call into slot history_slot(slot0, j, C).
struct HistoryAppend {
    long long src0;     // n16 - m
    int m;
    int slot0;          // (seen + n16 - m) mod C
};
MWW_HD HistoryAppend history_append_plan(long long seen, int n16, int C) {
    HistoryAppend p;
    p.m = n16 < C ? n16 : C;
    p.src0 = (long long)n16 - p.m;
    p.slot0 = history_mod(seen + p.src0, C);
    return p;
}

// A read of the last n samples (0 <= n <= C) after `seen`: entry k (oldest first) is in slot history_slot(slot0, k, C).  The
// run is at most two segments of the ring, [slot0, C) and [0, ...).
MWW_HD int history_read_slot0(long long seen, int n, int C) { return history_mod(seen - n, C); }

// 8-sample vectors, for the append: a call's units are the m / 8 vectors when every vector starts on a multiple of 8 in the
// ring (slot0 % 8 == 0) and in the caller's row (src0 % 8 == 0, row pitch % 8 == 0) and m % 8 == 0; the launcher adds the
// alignment of the row base (history_append_vec_ok in mww_history.cu).  Otherwise one sample per unit.
MWW_HD bool history_append_vec_shape(const HistoryAppend &p, long long audio_stride) {
    return p.slot0 % 8 == 0 && p.src0 % 8 == 0 && p.m % 8 == 0 && audio_stride % 8 == 0;
}
// likewise for a read of n samples into rows of pitch out_stride
MWW_HD bool history_read_vec_shape(int slot0, int n, long long out_stride) { return slot0 % 8 == 0 && n % 8 == 0 && out_stride % 8 == 0; }

// ---- per-element bodies of the two kernels (the device forms move 8 samples at once where the *_vec_shape tests pass) ----
// append: sample j of the call of one stream (its row of the caller's audio, and its ring row)
template <typename T>
MWW_HD void history_append_one(int16_t *ring_row, const T *audio_row, const HistoryAppend &p, int j, int C) {
    ring_row[history_slot(p.slot0, j, C)] = pcm16(audio_row[p.src0 + j]);
}
// read: entry k of row i of the output for stream id; an id outside [0, n_streams) reads as zeros
MWW_HD int16_t history_read_one(const int16_t *ring, int C, int id, int n_streams, int slot0, int k) {
    if (id < 0 || id >= n_streams) return 0;
    return ring[(long long)id * C + history_slot(slot0, k, C)];
}

// ---- the write (mww_write_audio_history; kernel in mww_serving_records.cu) ------------------------------------------------------
// A row of n samples written after `seen`: the stream's history becomes zeros followed by the row, so sample t of the row sits
// at axis position seen - n + t.  The ring holds positions [seen - C, seen); entry e (oldest first) of that window is
// position seen - C + e in slot history_slot(slot0, e, C), and holds row sample e - lead when that is >= 0, else zero.
// lead = C - n is negative when n > C: only the row's last C samples land.  Every entry of the row is written.
struct HistoryWrite {
    long long lead;
    int slot0;          // seen mod C
};
MWW_HD HistoryWrite history_write_plan(long long seen, int n, int C) {
    HistoryWrite p;
    p.lead = (long long)C - n;
    p.slot0 = history_mod(seen, C);
    return p;
}
// 8-entry units when every unit starts on a multiple of 8 in the ring and in the caller's row, so a unit is all zeros or all
// row samples; the launcher adds the 16-byte alignment of the caller's buffer
MWW_HD bool history_write_vec_shape(const HistoryWrite &p, long long in_stride) {
    return p.slot0 % 8 == 0 && p.lead % 8 == 0 && in_stride % 8 == 0;
}
// write: entry e of one stream's ring row from its row of the caller's samples
MWW_HD void history_write_one(int16_t *ring_row, const int16_t *in_row, const HistoryWrite &p, int e, int C) {
    const long long t = (long long)e - p.lead;
    ring_row[history_slot(p.slot0, e, C)] = t >= 0 ? in_row[t] : (int16_t)0;
}

}  // namespace mww
