"""What the positioned endpointer costs: one Endpointer.update over 65 536 rows with 1 and with 100 steps per call, on a plain
endpointer and on a positioned one (arm(ids, at=...)) whose rows are all armed with a running mute, the two arms alternating
round by round; and one positioned arm of 32, 1 024 and 4 096 slots (two launches: the reduction of each row's latest
position and the arm), beside a plain arm of the same ids.  From a 65 536-stream fp32 okay_nabu engine with an 8 s history.
Times in ms per call from CUDA events, the best of --rounds rounds; an update is timed one call at a time, with the
endpointer's baseline set back and its rows armed again (synchronously, outside the timed span) so that the same update fits
the engine's counters again.  Prints the card, its power limit and the SM clock sampled during the run.  There is no CPU
path: without a GPU it fails.
    python tools/endpoint_at_time.py [--streams 65536] [--slots 32 1024 4096] [--rounds 5]"""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench import ClockSampler, model_blob, synth_audio_device  # noqa: E402
from endpoint_time import HISTORY, P, card, event_time, set_baseline  # noqa: E402
from microwakeword_b200.endpoint import Endpointer  # noqa: E402
from microwakeword_b200.engine import StreamEngine  # noqa: E402


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--streams", type=int, default=65536)
    ap.add_argument("--slots", type=int, nargs="+", default=[32, 1024, 4096])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("endpoint_at_time.py measures the GPU kernels and needs a CUDA device; none is available")
    S = a.streams
    print("card: %s; %d streams, fp32 okay_nabu, history %d samples" % (card(), S, HISTORY))
    clocks = ClockSampler(0)
    times = {}
    try:
        eng = StreamEngine(model_blob("f32"), n_streams=S)
        eng.set_audio_history(HISTORY)
        idx = torch.arange(S, device="cuda") % P
        audio = synth_audio_device(torch, P, 480 * 80, 3, torch.device("cuda", 0))[idx].contiguous()
        plain = Endpointer(eng, lookback_steps=64, timeout_steps=1000, max_steps=1000)
        at = Endpointer(eng, lookback_steps=64, timeout_steps=1000, max_steps=1000)
        for i in range(240):                         # flags for the replays, and a baseline 100 steps can be set back from
            p = eng.step(audio[:, 480 * (i % 80):480 * (i % 80 + 1)])
            plain.update(p)
            at.update(p)
        info = eng._info()
        seen, buffered, pending = eng.audio_samples_seen, info.frontend_buffered, info.pending_rows
        every = torch.arange(S, dtype=torch.int32, device="cuda")
        q = seen - (buffered - (480 - plain.hop)) - plain.hop * pending
        newest = torch.full((S,), q, dtype=torch.int64, device="cuda")
        vad = torch.rand((S, 100), dtype=torch.float32, device="cuda")
        skip = 200 * plain.stride * plain.hop           # a mute that outlasts every timed update
        for n in (1, 100):
            pr = vad[:, :n]
            for rnd in range(a.rounds):
                for name, ep in (("plain", plain), ("positioned", at)):
                    def back(ep=ep, n=n):
                        set_baseline(ep, seen, buffered, pending)
                        if ep is at:
                            ep.arm(every, at=newest, skip=skip)
                        else:
                            ep.arm(every)
                        set_baseline(ep, seen - n * ep.stride * ep.hop, buffered, pending)
                    times.setdefault("update, %d step(s), every row armed, %s" % (n, name), []).append(
                        event_time(lambda ep=ep, pr=pr: ep.update(pr), a.calls, before=back))
        set_baseline(plain, seen, buffered, pending)
        set_baseline(at, seen, buffered, pending)
        gen = torch.Generator(device="cuda").manual_seed(0)
        for slots in a.slots:
            ids = torch.randperm(S, device="cuda", generator=gen)[:slots].to(torch.int32)
            pos = newest[:slots] - 480 * torch.randint(0, 60, (slots,), device="cuda", generator=gen)
            for rnd in range(a.rounds):
                times.setdefault("arm, %d slots, plain" % slots, []).append(event_time(lambda ids=ids: plain.arm(ids), a.calls))
                times.setdefault("arm, %d slots, positioned" % slots, []).append(
                    event_time(lambda ids=ids, pos=pos: at.arm(ids, at=pos), a.calls))
        print("positioned: %s, plain: %s; launches %d / %d" % (at.positioned, plain.positioned, at.launch_count, plain.launch_count))
    finally:
        sampled = clocks.stop()
    print("SM clock during the run: median %s MHz (max %s MHz), throttle reasons seen: %s" %
          (sampled["sm_mhz"], sampled["sm_max_mhz"], ", ".join(sampled["reasons"]) or "none"))
    for k, t in times.items():
        print("%-52s best %8.3f ms per call (rounds %s)" % (k, min(t), " / ".join("%.3f" % x for x in t)))


if __name__ == "__main__":
    main()
