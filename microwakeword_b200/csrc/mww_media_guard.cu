// mww_media_guard.cu -- the four kernels of the media guard (bodies: mww_media_guard.h; rule in include/mww.h, "media guard"):
// the slots of a check, fingerprints from feature rows, the (slot x candidate) lag search, and the decision with the ring
// append.  Each is one launch whatever the number of events.  A companion library of its own, libmww_media_guard.so, so that
// libmww_b200.so and the other companion libraries keep exactly the kernels they had.
#include <algorithm>

#include "mww_kernels.h"

namespace mww {

namespace {

constexpr int kSlotThreads = 1024;      // the slots kernel is one CTA: the ranks of the valid slots are a prefix count
constexpr int kFpThreads = 256;
constexpr int kMatchWarps = 8;
constexpr int kDecideThreads = 128;
constexpr unsigned kFull = 0xffffffffu;

// Slot i of the check (media_slot_detector with events, else media_slot_streams), its rank among the valid slots, and the
// ring state: base = the count before this check, total = its valid slots, count advanced by total.  Zeroes the counters the
// match kernel adds to.
__global__ void __launch_bounds__(kSlotThreads) media_slots_kernel(const MediaSlotsArgs a, const MediaSlotsOut o) {
    __shared__ int warp_total[kSlotThreads / 32];
    __shared__ long long carry;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) carry = 0;
    const long long count = a.events ? *a.count : 0;
    for (int first = 0; first < a.n; first += kSlotThreads) {
        const int i = first + tid;
        bool valid = false;
        if (i < a.n) {
            const MediaSlot s = a.events ? media_slot_detector(i, count, a.capacity, a.events, a.positions, a.ev_group, a.model, a.post, a.seen,
                                                               a.C, a.n_samples)
                                         : media_slot_streams(a.ids[i], a.ends[i], a.households ? a.households[i] : -1, a.n_streams, a.seen,
                                                              a.C, a.n_samples);
            o.sid[i] = s.sid; o.rid[i] = s.rid; o.hh[i] = s.hh; o.end[i] = s.end; o.pos[i] = s.pos;
            o.count[i] = 0; o.clip_hit[i] = 0;
            valid = s.rid >= 0;
        }
        const unsigned ballot = __ballot_sync(kFull, valid);
        if (lane == 0) warp_total[warp] = __popc(ballot);
        __syncthreads();
        int before = 0, chunk = 0;
        for (int w = 0; w < kSlotThreads / 32; ++w) {
            before += w < warp ? warp_total[w] : 0;
            chunk += warp_total[w];
        }
        if (i < a.n) o.rank[i] = valid ? (int32_t)(carry + before + __popc(ballot & ((1u << lane) - 1u))) : -1;
        __syncthreads();
        if (tid == 0) carry += chunk;
        __syncthreads();
    }
    if (tid == 0) {
        MediaRingState s = *o.state;
        s.base = s.count;
        s.total = carry;
        s.count += carry;
        *o.state = s;
    }
}

// word t of row s: fp[s][t] from feature rows t and t + 1 of feat [n][rows][40]
__global__ void __launch_bounds__(kFpThreads) media_fingerprint_kernel(const uint16_t *__restrict__ feat, long long rows, int n, int words,
                                                                      uint64_t *__restrict__ fp, long long fp_stride) {
    const long long k = (long long)blockIdx.x * kFpThreads + threadIdx.x;
    if (k >= (long long)n * words) return;
    const long long s = k / words, t = k % words;
    const uint16_t *r = feat + (s * rows + t) * kNumChannels;
    fp[s * fp_stride + t] = media_fp_word(r, r + kNumChannels);
}

// CTA (i, y): slot i's fingerprint in shared memory, and the candidate tasks [y T, (y + 1) T), T = a.tasks_per_cta, a warp each:
// this check's slots [0, n), the ring's entries [n, n + ring), then the registered clips' lag chunks.  A task that passes the
// household and window filters stages its candidate's words in the warp's shared buffer, and the lanes take its lags.
__global__ void __launch_bounds__(kMatchWarps * 32) media_match_kernel(const MediaMatchArgs a) {
    extern __shared__ uint64_t smem[];
    const int i = blockIdx.x, W = a.words;
    const int32_t s_i = a.rid[i];
    if (s_i < 0) return;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint64_t *xs = smem, *buf = smem + W + warp * (W + kMediaLagChunk);
    for (int t = threadIdx.x; t < W; t += kMatchWarps * 32) xs[t] = a.fp[(long long)i * W + t];
    __syncthreads();
    const int32_t h_i = a.hh[i];
    const long long p_i = a.pos[i];
    const long long fill = a.ring > 0 ? (a.state->base < a.ring ? a.state->base : a.ring) : 0;
    const long long first = (long long)blockIdx.y * a.tasks_per_cta;
    for (int w = warp; w < a.tasks_per_cta; w += kMatchWarps) {
        const long long j = first + w;
        const uint64_t *src;
        int ny = W, y_base = 0, lo = -a.max_lag, hi = a.max_lag;
        bool clip = false;
        if (j < a.n) {
            const int32_t s_j = a.rid[j];
            if (j == i || s_j < 0 || !media_candidate(h_i, s_i, p_i, a.hh[j], s_j, a.pos[j], a.window)) continue;
            src = a.fp + j * W;
        } else if (j < a.n + a.ring) {
            const long long r = j - a.n;
            if (r >= fill || !media_candidate(h_i, s_i, p_i, a.ring_hh[r], a.ring_stream[r], a.ring_pos[r], a.window)) continue;
            src = a.ring_fp + r * W;
        } else {
            const long long q = j - a.n - a.ring;
            if (q >= a.clip_tasks) continue;
            int k = 0;
            for (int step = 1 << 12; step; step >>= 1)        // the last clip whose first task is <= q (at most 4096 clips)
                if (k + step < a.n_clips && a.clip_task0[k + step] <= q) k += step;
            ny = a.clip_len[k];
            lo = media_lag_lo(W, a.min_overlap) + (int)(q - a.clip_task0[k]) * kMediaLagChunk;
            const int top = media_lag_hi(ny, a.min_overlap);
            hi = lo + kMediaLagChunk - 1 < top ? lo + kMediaLagChunk - 1 : top;
            y_base = lo > 0 ? lo : 0;
            src = a.clip_fp + a.clip_off[k];
            clip = true;
        }
        const int y_end = ny < W + hi ? ny : W + hi;
        for (int u = lane; u < y_end - y_base; u += 32) buf[u] = src[y_base + u];
        __syncwarp();
        bool ok = false;
        for (int l = lo + lane; l <= hi && !ok; l += 32) ok = media_lag_matches(xs, W, buf, y_base, ny, l, a.min_overlap, a.max_ber_milli);
        if (__any_sync(kFull, ok) && lane == 0) {
            if (clip) atomicOr(&a.clip_hit[i], 1);
            else atomicAdd(&a.count[i], 1);
        }
        __syncwarp();
    }
}

// slot i: matches, media and passed (media_decide), and its ring entry (media_ring_entry) when it is valid
__global__ void __launch_bounds__(kDecideThreads) media_decide_kernel(const MediaDecideArgs a) {
    const int i = blockIdx.x;
    const int32_t rid = a.rid[i];
    if (threadIdx.x == 0) {
        const MediaOut o = media_decide(rid >= 0, a.count[i], a.clip_hit[i], a.min_matches, a.confirmed ? a.confirmed[i] : a.sid[i]);
        if (a.matches) a.matches[i] = o.matches;
        if (a.media) a.media[i] = o.media;
        if (a.passed) a.passed[i] = o.passed;
    }
    if (rid < 0) return;
    const MediaRingState s = *a.state;
    const long long e = media_ring_entry(s.base, s.total, a.rank[i], a.ring);
    if (e < 0) return;
    for (int t = threadIdx.x; t < a.words; t += kDecideThreads) a.ring_fp[e * a.words + t] = a.fp[(long long)i * a.words + t];
    if (threadIdx.x == 0) {
        a.ring_stream[e] = rid;
        a.ring_hh[e] = a.hh[i];
        a.ring_pos[e] = a.pos[i];
    }
}

}  // namespace

size_t media_match_smem(int words) { return (size_t)(words + kMatchWarps * (words + kMediaLagChunk)) * sizeof(uint64_t); }

cudaError_t launch_media_slots(const MediaSlotsArgs &a, const MediaSlotsOut &o, cudaStream_t st) {
    media_slots_kernel<<<1, kSlotThreads, 0, st>>>(a, o);
    return cudaGetLastError();
}

cudaError_t launch_media_fingerprint(const uint16_t *feat, long long rows, int n, int words, uint64_t *fp, long long fp_stride, cudaStream_t st) {
    const long long total = (long long)n * words;
    if (total <= 0) return cudaSuccess;
    media_fingerprint_kernel<<<(unsigned)((total + kFpThreads - 1) / kFpThreads), kFpThreads, 0, st>>>(feat, rows, n, words, fp, fp_stride);
    return cudaGetLastError();
}

cudaError_t launch_media_match(const MediaMatchArgs &a, cudaStream_t st) {
    // the opt-in is per device and not per guard: opt into what the longest clip any rule allows needs, so that a guard with
    // a longer clip than the first one launched on this device still fits
    static bool done[64] = {};
    const size_t smem = media_match_smem(a.words), most = media_match_smem(kMediaMaxWords);
    if (most > 48 * 1024 && first_launch_on_this_device(done))
        if (cudaError_t e = cudaFuncSetAttribute(media_match_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)most)) return e;
    // 8 tasks per warp, or more when the tasks would need more than 65 535 CTAs in y
    const long long tasks = a.n + a.ring + a.clip_tasks;
    MediaMatchArgs b = a;
    const long long per = std::max<long long>(8 * kMatchWarps, (tasks + 65534) / 65535);
    b.tasks_per_cta = (int)((per + kMatchWarps - 1) / kMatchWarps * kMatchWarps);
    const long long y = (tasks + b.tasks_per_cta - 1) / b.tasks_per_cta;
    if (a.n <= 0 || y <= 0) return cudaSuccess;
    media_match_kernel<<<dim3((unsigned)a.n, (unsigned)y), kMatchWarps * 32, smem, st>>>(b);
    return cudaGetLastError();
}

cudaError_t launch_media_decide(const MediaDecideArgs &a, cudaStream_t st) {
    if (a.n <= 0) return cudaSuccess;
    media_decide_kernel<<<(unsigned)a.n, kDecideThreads, 0, st>>>(a);
    return cudaGetLastError();
}

}  // namespace mww
