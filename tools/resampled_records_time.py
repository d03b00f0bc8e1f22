"""What moving resampled streams costs: export and import (mww_export_resampled_streams / mww_import_resampled_streams) of
--streams streams of an fp32 okay_nabu engine at 48 kHz, of one with per-stream rates (all seven rates in turn), and of a
plain 16 kHz engine, there beside the same move with the stream records alone (mww_export_streams / mww_import_streams).
Beside them one 480-sample step() (1 440 samples) of the 48 kHz engine.  Times in ms per call from CUDA events, the best of
--rounds rounds.  Prints the card, its power limit and the SM clock sampled during the run.  There is no CPU path: without
a GPU it fails.
    python tools/resampled_records_time.py [--streams 65536] [--rounds 5]"""
import argparse
import ctypes
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import ClockSampler, model_blob  # noqa: E402
from microwakeword_b200 import _lib  # noqa: E402
from microwakeword_b200.engine import INPUT_RATES, StreamEngine  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "%s (nvidia-smi unavailable)" % torch.cuda.get_device_name(0)


def event_time(fn, calls):
    fn()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(calls):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / calls


def warm(eng, S, per_stream):
    """ten 30 ms calls of noise, so that every history and ring holds data"""
    g = torch.Generator(device="cuda").manual_seed(1)
    for _ in range(10):
        if per_stream:
            width = int(eng.inputs_for(480).max())
            eng.step(torch.randint(-3000, 3000, (S, width), dtype=torch.int16, device="cuda", generator=g))
        else:
            n = {48000: 1440, 16000: 480}[eng.input_rate]
            eng.step(torch.randint(-3000, 3000, (S, n), dtype=torch.int16, device="cuda", generator=g))


def move(eng, S, resampler):
    """export and import of every stream into its own slot, records preallocated: -> (export, import, record bytes)"""
    L, h = eng._L, eng._h
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    ids = np.random.default_rng(0).permutation(S).astype(np.int32)
    lay, rs = _lib.MwwStreamLayout(), _lib.MwwResamplerLayout()
    rates = np.zeros(S, np.int32)
    if resampler:
        rec = torch.empty((S, int(eng.resampler_layout().record_bytes)), dtype=torch.uint8, device="cuda")

        def exp():
            _lib.check(h, L.mww_export_resampled_streams(h, ids.ctypes.data, S, rec.data_ptr(), ctypes.byref(lay), ctypes.byref(rs),
                                                         rates.ctypes.data, st))

        def imp():
            _lib.check(h, L.mww_import_resampled_streams(h, ids.ctypes.data, S, rec.data_ptr(), ctypes.byref(lay), ctypes.byref(rs),
                                                         rates.ctypes.data, st))
    else:
        rec = torch.empty((S, int(eng.stream_layout().record_bytes)), dtype=torch.uint8, device="cuda")

        def exp():
            _lib.check(h, L.mww_export_streams(h, ids.ctypes.data, S, rec.data_ptr(), ctypes.byref(lay), st))

        def imp():
            _lib.check(h, L.mww_import_streams(h, ids.ctypes.data, S, rec.data_ptr(), ctypes.byref(lay), st))
    exp()
    return exp, imp, rec.shape[1]


def timed(times, label, eng, S, resampler, a):
    exp, imp, rb = move(eng, S, resampler)
    times["%s: export (%d B records)" % (label, rb)] = [event_time(exp, a.calls) for _ in range(a.rounds)]
    times["%s: import" % label] = [event_time(imp, a.calls) for _ in range(a.rounds)]


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--streams", type=int, default=65536)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("resampled_records_time.py measures the GPU kernels and needs a CUDA device; none is available")
    S = a.streams
    print("card: %s; %d streams, fp32 okay_nabu" % (card(), S))
    clocks = ClockSampler(0)
    times = {}
    try:
        blob = model_blob("f32")
        eng = StreamEngine(blob, n_streams=S)
        eng.set_input_rate(48000)
        warm(eng, S, False)
        chunk = torch.randint(-3000, 3000, (S, 1440), dtype=torch.int16, device="cuda")
        probs = torch.empty((S, 1), dtype=torch.float32, device="cuda")
        times["step() 1 440 samples at 48 kHz"] = [event_time(lambda: eng.step(chunk, out=probs), 50) for _ in range(a.rounds)]
        timed(times, "48 kHz, resampled", eng, S, True, a)
        del eng
        eng = StreamEngine(blob, n_streams=S)
        eng.set_stream_rates(np.arange(S), np.asarray(INPUT_RATES, np.int32)[np.arange(S) % len(INPUT_RATES)])
        warm(eng, S, True)
        timed(times, "per-stream rates, resampled", eng, S, True, a)
        del eng
        eng = StreamEngine(blob, n_streams=S)
        warm(eng, S, False)
        timed(times, "16 kHz, resampled", eng, S, True, a)
        timed(times, "16 kHz, stream records", eng, S, False, a)
    finally:
        sampled = clocks.stop()
    print("SM clock during the run: median %s MHz (max %s MHz), throttle reasons seen: %s" %
          (sampled["sm_mhz"], sampled["sm_max_mhz"], ", ".join(sampled["reasons"]) or "none"))
    for k, t in times.items():
        print("%-56s best %8.3f ms per call (rounds %s)" % (k, min(t), " / ".join("%.3f" % x for x in t)))


if __name__ == "__main__":
    main()
