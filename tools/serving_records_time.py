"""What moving a stream's serving state costs: endpointer export and import (mww_export_endpointer_rows /
mww_import_endpointer_rows) at 1, 1 024 and 65 536 streams, and a history write (mww_write_audio_history) of 32 000 samples
for 1 024 and 65 536 streams, each beside torch.Tensor.copy_ of the same bytes on the same device, and one 480-sample step()
of the 65 536-stream fp32 okay_nabu engine the state belongs to.  Times in ms per call from CUDA events, the best of
--rounds rounds.  Prints the card, its power limit and the SM clock sampled during the run.  There is no CPU path: without
a GPU it fails.
    python tools/serving_records_time.py [--streams 65536] [--rounds 5]"""
import argparse
import ctypes
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import ClockSampler, model_blob, synth_audio_device  # noqa: E402
from microwakeword_b200 import _lib  # noqa: E402
from microwakeword_b200.endpoint import Endpointer  # noqa: E402
from microwakeword_b200.engine import StreamEngine  # noqa: E402

P = 1021                         # distinct base streams; stream s carries base[s % P]
HISTORY = 32000                  # 2 s


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


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--streams", type=int, default=65536)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("serving_records_time.py measures the GPU kernels and needs a CUDA device; none is available")
    S = a.streams
    print("card: %s; %d streams, fp32 okay_nabu, history %d samples" % (card(), S, HISTORY))
    clocks = ClockSampler(0)
    times = {}
    try:
        eng = StreamEngine(model_blob("f32"), n_streams=S)
        eng.set_audio_history(HISTORY)
        idx = torch.arange(S, device="cuda") % P
        audio = synth_audio_device(torch, P, 480 * 80, 3, torch.device("cuda", 0))[idx].contiguous()
        probs = torch.empty((S, 1), dtype=torch.float32, device="cuda")
        ep = Endpointer(eng, lookback_steps=64)
        for i in range(80):
            ep.update(eng.step(audio[:, 480 * i:480 * (i + 1)], out=probs))
            if i == 40:
                ep.arm(list(range(0, S, 2)))         # half the rows armed, so the records carry segmenter state
        chunk = audio[:, :480].contiguous()
        times["step() 480 samples, %d streams" % S] = [event_time(lambda: eng.step(chunk, out=probs), 50) for _ in range(a.rounds)]
        # the timed step() calls moved the engine on without updates: export and import need an endpointer that is up to date
        # with its engine, so a whole reset takes the engine's counters as the new baseline; re-arm half the rows
        ep.reset()
        ep.arm(list(range(0, S, 2)))
        L = eng._L
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        rb = int(ep.layout().record_bytes)
        lay = _lib.MwwEndpointerLayout()
        for n in (1, 1024, S):
            ids = torch.randperm(S)[:n].to(torch.int32).numpy()
            rec = torch.empty((n, rb), dtype=torch.uint8, device="cuda")
            twin = torch.empty_like(rec)
            exp = (lambda ids=ids, rec=rec: ep._check(L.mww_export_endpointer_rows(ep._ep, ids.ctypes.data, ids.size, rec.data_ptr(),
                                                                                 ctypes.byref(lay), st)))
            exp()
            imp = (lambda ids=ids, rec=rec: ep._check(L.mww_import_endpointer_rows(ep._ep, ids.ctypes.data, ids.size, rec.data_ptr(),
                                                                                 ctypes.byref(lay), st)))
            times["endpointer export, %d rows (%d B each)" % (n, rb)] = [event_time(exp, a.calls) for _ in range(a.rounds)]
            times["endpointer import, %d rows" % n] = [event_time(imp, a.calls) for _ in range(a.rounds)]
            times["copy_ of the same %d bytes" % (n * rb)] = [event_time(lambda t=twin, r=rec: t.copy_(r), a.calls) for _ in range(a.rounds)]
        for n in (1024, S):
            ids = torch.randperm(S)[:n].to(torch.int32).numpy()
            rows = torch.randint(-3000, 3000, (n, HISTORY), dtype=torch.int16, device="cuda")
            twin = torch.empty_like(rows)
            wr = (lambda ids=ids, rows=rows: _lib.check(eng._h, L.mww_write_audio_history(eng._h, ids.ctypes.data, ids.size, HISTORY,
                                                                                        rows.data_ptr(), HISTORY, st)))
            times["history write, %d streams x %d samples" % (n, HISTORY)] = [event_time(wr, a.calls) for _ in range(a.rounds)]
            times["copy_ of the same %d bytes" % (2 * n * HISTORY)] = [event_time(lambda t=twin, r=rows: t.copy_(r), a.calls)
                                                                      for _ in range(a.rounds)]
            del rows, twin
    finally:
        sampled = clocks.stop()
    print("SM clock during the run: median %s MHz (max %s MHz), throttle reasons seen: %s" %
          (sampled["sm_mhz"], sampled["sm_max_mhz"], ", ".join(sampled["reasons"]) or "none"))
    for k, t in times.items():
        print("%-48s best %8.3f ms per call (rounds %s)" % (k, min(t), " / ".join("%.3f" % x for x in t)))


if __name__ == "__main__":
    main()
