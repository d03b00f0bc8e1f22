// tests/emul_endpoint.cc -- TEST INFRASTRUCTURE: the per-row bodies of the endpointer's kernels
// (microwakeword_b200/csrc/mww_endpoint.h) run on the CPU, a row or an id at a time as the kernels' threads run them, for
// tests/test_endpoint.py.  Never used by the product.
#include "../microwakeword_b200/csrc/mww_endpoint.h"

using namespace mww;

namespace {
// cfg: vad_window, speech_steps, silence_steps, timeout_steps, max_steps, lookback_steps, n_rows, n_streams, capacity;
// p: hist, seen, flags, armed, elapsed, run, silence, heard, start, speech_end, arm_tag, row_of, count, events, ended
EndpointArgs args(const int *cfg, double cutoff, long long step_samples, void **p) {
    EndpointArgs a;
    a.rule = mww_endpoint_rule{cfg[0], cfg[1], cfg[2], cfg[3], cfg[4], cfg[5], cutoff};
    a.n_rows = cfg[6]; a.n_streams = cfg[7]; a.capacity = cfg[8];
    a.step_samples = step_samples;
    a.hist = (float *)p[0]; a.seen = (long long *)p[1]; a.flags = (unsigned long long *)p[2]; a.armed = (int32_t *)p[3];
    a.elapsed = (int32_t *)p[4]; a.run = (int32_t *)p[5]; a.silence = (int32_t *)p[6]; a.heard = (int32_t *)p[7];
    a.start = (long long *)p[8]; a.speech_end = (long long *)p[9]; a.arm_tag = (int32_t *)p[10]; a.row_of = (const int32_t *)p[11];
    a.count = (unsigned long long *)p[12]; a.events = (mww_endpoint_event *)p[13]; a.ended = (int32_t *)p[14];
    return a;
}
}  // namespace

extern "C" void emul_endpoint_update(const int *cfg, double cutoff, long long step_samples, void **p, const float *probs, long long pitch,
                                     int n, long long pos0) {
    const EndpointArgs a = args(cfg, cutoff, step_samples, p);
    for (int r = 0; r < a.n_rows; ++r) endpoint_update_row(a, r, probs, pitch, n, pos0);
}

extern "C" void emul_endpoint_arm(const int *cfg, double cutoff, long long step_samples, void **p, const int32_t *ids, int n, int steps,
                                  int tag, const long long *pos) {
    const EndpointArgs a = args(cfg, cutoff, step_samples, p);
    EndpointReplay R;
    R.steps = steps; R.tag = tag;
    for (int i = 0; i < kEndpointMaxLookback; ++i) R.pos[i] = pos[i];
    for (int i = 0; i < n; ++i) endpoint_arm_one(a, R, ids[i]);
}

extern "C" void emul_endpoint_clear(const int *cfg, double cutoff, long long step_samples, void **p, const int32_t *ids, int n, int reset) {
    const EndpointArgs a = args(cfg, cutoff, step_samples, p);
    for (int i = 0; i < n; ++i) {
        const int r = ids ? endpoint_row(a, ids[i]) : i;
        if (r >= 0) endpoint_clear_row(a, r, reset);
    }
}

extern "C" long long emul_endpoint_position(long long S, int buffered, int hop, int pending, int stride, int n, int j) {
    return endpoint_position(S, buffered, hop, pending, stride, n, j);
}

extern "C" int emul_endpoint_fits(long long S0, int buffered0, int pending0, long long S, int buffered, int pending, int hop, int stride, int n) {
    return endpoint_update_fits(S0, buffered0, pending0, S, buffered, pending, hop, stride, n);
}

// the command read, a sample at a time: out [capacity][out_stride], lengths [capacity]
extern "C" void emul_endpoint_read(const int16_t *ring, int C, long long seen, long long count, const mww_endpoint_event *events, int capacity,
                                   long long pre, long long post, int max_samples, int16_t *out, long long out_stride, int32_t *lengths) {
    for (int i = 0; i < capacity; ++i) {
        const CommandSpan c = endpoint_command_span(i, count, capacity, events, pre, post, max_samples);
        lengths[i] = c.len;
        for (int k = 0; k < max_samples; ++k)
            out[(long long)i * out_stride + k] = k < c.len ? endpoint_command_one(ring, C, seen, events[i].stream, c.a + k) : (int16_t)0;
    }
}
