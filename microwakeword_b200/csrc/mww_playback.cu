// mww_playback.cu -- the three kernels of the playback guard (bodies: mww_playback.h; rule in include/mww.h, "playback guard"):
// the write of a call's rows, the slots of a check with the read of their reference clips (also the public read), and the
// decision.  Each is one launch whatever the number of rows or events.  A companion library of its own, libmww_playback.so, so
// that libmww_b200.so and the other companion libraries keep exactly the kernels they had.
#include "mww_kernels.h"

namespace mww {

namespace {

constexpr int kWriteThreads = 128;
constexpr int kReadThreads = 256;
constexpr int kDecideThreads = 128;

// CTA j: job j of a write call.  A job with a row writes row j of the caller's audio (8-sample units where
// playback_write_vec_shape holds and vec_base is set); one without (row -1) only clears its stream's map entry.  Thread 0 updates
// the map and the head, which no other thread of the launch reads.
__global__ void __launch_bounds__(kWriteThreads)
playback_write_kernel(const PlaybackJob *__restrict__ jobs, const int16_t *__restrict__ audio, long long audio_stride, int n_samples,
                      int vec_base, int16_t *__restrict__ ring, int C, int32_t *__restrict__ row_of, long long *__restrict__ head) {
    const PlaybackJob job = jobs[blockIdx.x];
    if (job.row < 0) {
        if (threadIdx.x == 0) row_of[job.stream] = -1;
        return;
    }
    const PlaybackWrite p = playback_write_plan(job.start, n_samples, job.head, C);
    int16_t *row = ring + (long long)job.row * C;
    const int16_t *x = audio + (long long)blockIdx.x * audio_stride;
    if (vec_base && playback_write_vec_shape(p, job.start, n_samples, audio_stride)) {
        for (long long u = threadIdx.x; u < p.len / 8; u += kWriteThreads) {
            const long long q = p.span0 + 8 * u;
            const uint4 v = q < job.start ? make_uint4(0, 0, 0, 0) : *reinterpret_cast<const uint4 *>(x + (q - job.start));
            *reinterpret_cast<uint4 *>(row + playback_mod(q, C)) = v;
        }
    } else {
        for (long long k = threadIdx.x; k < p.len; k += kWriteThreads) {
            const long long q = p.span0 + k;
            row[playback_mod(q, C)] = playback_write_value(x, job.start, q);
        }
    }
    if (threadIdx.x == 0) {
        row_of[job.stream] = job.row;
        head[job.row] = p.head;
    }
}

// CTA i: slot i (playback_slot_detector with events, else playback_slot_streams), and the read of pb over [r1 - L, r1),
// r1 = e - a.min_delay, into out row i: 8-entry units (16-byte loads from the ring where the unit lies inside [w - C, w))
// when a.vec.  With a.sid set (a check), thread 0 also writes the slot's stream and whether it is heard.
__global__ void __launch_bounds__(kReadThreads) playback_slots_kernel(const PlaybackSlotsArgs a) {
    const int i = blockIdx.x;
    const PlaybackSlot s = a.events ? playback_slot_detector(i, *a.count, a.capacity, a.events, a.positions, a.model, a.post, a.seen)
                                    : playback_slot_streams(a.ids[i], a.ends[i]);
    const bool listed = s.sid >= 0 && s.sid < a.n_streams;
    const int32_t r = listed ? a.row_of[s.sid] : -1;
    const bool has_row = r >= 0;
    const long long w = has_row ? a.head[r] : 0;
    const long long r1 = playback_ref_end(s.end, a.min_delay), r0 = r1 - a.L;
    if (a.sid && threadIdx.x == 0) {
        a.sid[i] = s.sid;
        a.heard[i] = playback_heard(s.sid, a.n_streams, has_row, w, r0, a.seen, a.C) ? 1 : 0;
    }
    const int16_t *row = a.ring + (long long)(has_row ? r : 0) * a.C;
    int16_t *dst = a.out + (long long)i * a.out_stride;
    if (a.vec && playback_mod(r0, 8) == 0) {
        for (int u = threadIdx.x; u < a.L / 8; u += kReadThreads) {
            const long long q = r0 + 8 * u;
            uint4 v = make_uint4(0, 0, 0, 0);
            if (has_row && playback_held(q, w, a.C) && playback_held(q + 7, w, a.C)) {
                v = *reinterpret_cast<const uint4 *>(row + playback_mod(q, a.C));
            } else if (has_row && (playback_held(q, w, a.C) || playback_held(q + 7, w, a.C))) {
                int16_t e[8];
#pragma unroll
                for (int k = 0; k < 8; ++k) e[k] = playback_read_one(row, a.C, true, w, q + k);
                v = make_uint4(pack16(e[0], e[1]), pack16(e[2], e[3]), pack16(e[4], e[5]), pack16(e[6], e[7]));
            }
            *reinterpret_cast<uint4 *>(dst + 8 * u) = v;
        }
    } else {
        for (int k = threadIdx.x; k < a.L; k += kReadThreads) dst[k] = playback_read_one(row, a.C, has_row, w, r0 + k);
    }
}

__global__ void __launch_bounds__(kDecideThreads)
playback_decide_kernel(int n, const int32_t *__restrict__ sid, const int32_t *__restrict__ heard, const float *__restrict__ scores, double cutoff,
                       const int32_t *__restrict__ confirmed, float *__restrict__ out_scores, int32_t *__restrict__ out_flagged,
                       int32_t *__restrict__ out_passed) {
    const int i = blockIdx.x * kDecideThreads + threadIdx.x;
    if (i >= n) return;
    const PlaybackOut o = playback_decide(heard[i] != 0, scores[i], cutoff, confirmed ? confirmed[i] : sid[i]);
    if (out_scores) out_scores[i] = o.score;
    if (out_flagged) out_flagged[i] = o.flagged;
    if (out_passed) out_passed[i] = o.passed;
}

}  // namespace

cudaError_t launch_playback_write(const PlaybackJob *jobs, int n_jobs, const int16_t *audio, long long audio_stride, int n_samples,
                                  int16_t *ring, int C, int32_t *row_of, long long *head, cudaStream_t st) {
    if (n_jobs <= 0) return cudaSuccess;
    const int vec_base = reinterpret_cast<uintptr_t>(audio) % 16 == 0;
    playback_write_kernel<<<(unsigned)n_jobs, kWriteThreads, 0, st>>>(jobs, audio, audio_stride, n_samples, vec_base, ring, C, row_of, head);
    return cudaGetLastError();
}

cudaError_t launch_playback_slots(const PlaybackSlotsArgs &a, cudaStream_t st) {
    if (a.n <= 0) return cudaSuccess;
    PlaybackSlotsArgs b = a;
    b.vec = a.L % 8 == 0 && a.out_stride % 8 == 0 && reinterpret_cast<uintptr_t>(a.out) % 16 == 0;
    playback_slots_kernel<<<(unsigned)a.n, kReadThreads, 0, st>>>(b);
    return cudaGetLastError();
}

cudaError_t launch_playback_decide(int n, const int32_t *sid, const int32_t *heard, const float *scores, double cutoff, const int32_t *confirmed,
                                   float *out_scores, int32_t *out_flagged, int32_t *out_passed, cudaStream_t st) {
    if (n <= 0) return cudaSuccess;
    playback_decide_kernel<<<(unsigned)((n + kDecideThreads - 1) / kDecideThreads), kDecideThreads, 0, st>>>(n, sid, heard, scores, cutoff, confirmed,
                                                                                                           out_scores, out_flagged, out_passed);
    return cudaGetLastError();
}

}  // namespace mww
