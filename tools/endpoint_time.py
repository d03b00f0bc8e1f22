"""What endpointing costs: one Endpointer.update over 65 536 rows with 1 and with 100 steps per call, with no row armed and
with every row armed (the default rule: the segmenter on every row, and NO_SPEECH events at 100 steps), and one
Endpointer.commands read of 8 s clips (128 000 samples) at 64, 256 and 1 024 used event slots, from a 65 536-stream fp32
okay_nabu engine with an 8 s audio history.  Printed beside one 480-sample step() of the same engine.  Times in ms per call
from CUDA events, the best of --rounds rounds; an update is timed one call at a time, with the endpointer's baseline set
back (synchronously, outside the timed span) so that the same update fits the engine's counters again.  Prints the card, its
power limit and the SM clock sampled during the run.  There is no CPU path: without a GPU it fails.
    python tools/endpoint_time.py [--streams 65536] [--slots 64 256 1024] [--rounds 5]"""
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
HISTORY = 128000                 # 8 s
CLIP = 128000


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "%s (nvidia-smi unavailable)" % torch.cuda.get_device_name(0)


def event_time(fn, calls, before=None):
    total = 0.0
    for _ in range(calls):
        if before:
            before()
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        fn()
        end.record()
        end.synchronize()
        total += start.elapsed_time(end)
    return total / calls


def set_baseline(ep, seen, buffered, pending):
    """the endpointer's baseline counters only (NULL row arrays are skipped)"""
    st = _lib.MwwEndpointState()
    ep._check(ep._L.mww_endpointer_get_state(ep._ep, ctypes.byref(st)))
    st.samples_seen, st.buffered, st.pending = seen, buffered, pending
    ep._check(ep._L.mww_endpointer_set_state(ep._ep, ctypes.byref(st)))


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--streams", type=int, default=65536)
    ap.add_argument("--slots", type=int, nargs="+", default=[64, 256, 1024])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("endpoint_time.py measures the GPU kernels and needs a CUDA device; none is available")
    S = a.streams
    print("card: %s; %d streams, fp32 okay_nabu, history %d samples" % (card(), S, HISTORY))
    clocks = ClockSampler(0)
    times = {}
    try:
        eng = StreamEngine(model_blob("f32"), n_streams=S)
        eng.set_audio_history(HISTORY)
        idx = torch.arange(S, device="cuda") % P
        audio = synth_audio_device(torch, P, HISTORY + 480, 3, torch.device("cuda", 0))[idx].contiguous()
        probs = torch.empty((S, 1), dtype=torch.float32, device="cuda")
        ep = Endpointer(eng, capacity=max(a.slots), timeout_steps=1, lookback_steps=1)
        for i in range(HISTORY // 480):            # fill the history
            ep.update(eng.step(audio[:, 480 * i:480 * (i + 1)]))
        chunk = audio[:, :480].contiguous()
        times["step() 480 samples"] = [event_time(lambda: eng.step(chunk, out=probs), 50) for _ in range(a.rounds)]
        ep.reset()                                  # the engine moved on: take its counters again
        info = eng._info()
        seen, buffered, pending = eng.audio_samples_seen, info.frontend_buffered, info.pending_rows
        vad = torch.rand((S, 100), dtype=torch.float32, device="cuda")
        for n in (1, 100):
            p = vad[:, :n]
            back = (lambda n=n: set_baseline(ep, seen - n * ep.stride * ep.hop, buffered, pending))
            times["update, %d step(s), none armed" % n] = [event_time(lambda p=p: ep.update(p), a.calls, before=back) for _ in range(a.rounds)]
        # every row armed afresh before each timed update (outside the timed span), the default rule: the segmenter runs on
        # every row and step, and at 100 steps every row that heard no speech ends (NO_SPEECH) through the event counter
        epa = Endpointer(eng, lookback_steps=0, capacity=max(a.slots))
        every = torch.arange(S, dtype=torch.int32, device="cuda")
        for n in (1, 100):
            p = vad[:, :n]

            def back(n=n):
                set_baseline(epa, seen - n * epa.stride * epa.hop, buffered, pending)
                epa.drain()
                epa.arm(every)
            times["update, %d step(s), every row armed" % n] = [event_time(lambda p=p: epa.update(p), a.calls, before=back)
                                                               for _ in range(a.rounds)]
        print("events of the last armed 100-step update: %d" % int(epa.event_count.item()))
        epa.close()
        gen = torch.Generator(device="cuda").manual_seed(0)
        for slots in a.slots:
            # an endpointer of `slots` event slots, every slot used: each armed stream ends on its replayed step
            ep = Endpointer(eng, capacity=slots, timeout_steps=1, lookback_steps=1)
            eng.step(chunk, out=probs)
            ep.update(probs)
            ep.arm(torch.randperm(S, device="cuda", generator=gen)[:slots].to(torch.int32))
            assert int(ep.event_count.item()) == slots
            out = torch.empty((slots, CLIP), dtype=torch.int16, device="cuda")
            lengths = torch.empty(slots, dtype=torch.int32, device="cuda")
            fn = (lambda ep=ep, o=out, l=lengths: ep.commands(pre=CLIP, post=0, max_samples=CLIP, out=o, lengths=l))
            fn()
            times["commands, %d slots of %d samples" % (slots, CLIP)] = [event_time(fn, a.calls) for _ in range(a.rounds)]
            del out
            ep.close()
    finally:
        sampled = clocks.stop()
    print("SM clock during the run: median %s MHz (max %s MHz), throttle reasons seen: %s" %
          (sampled["sm_mhz"], sampled["sm_max_mhz"], ", ".join(sampled["reasons"]) or "none"))
    for k, t in times.items():
        print("%-44s best %8.3f ms per call (rounds %s)" % (k, min(t), " / ".join("%.3f" % x for x in t)))


if __name__ == "__main__":
    main()
