"""What the playback guard costs: on a 65 536-stream fp32 okay_nabu engine with a 48 000-sample audio history and a guard of
4 096 rows of 10 s, n_samples 24 000 and delays 0..16 000 (L_ref = 40 000), the time of
  * one PlaybackGuard.play of 4 096 playing rows x 480 samples (the real-time write of one poll), rows already held;
  * one PlaybackGuard.check (mww_playback_check_streams) of 32 and of 1 024 events, every event heard;
printed beside a 480-sample live step() of the same engine.  Times in ms per call from CUDA events, the best of --rounds rounds.
Prints the card, its power limit and the SM clock sampled during the run.  There is no CPU path: without a GPU it fails.
    python tools/playback_guard_time.py [--streams 65536] [--rounds 5] [--calls 10]"""
import argparse
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import ClockSampler, model_blob, synth_audio_device  # noqa: E402
from microwakeword_b200.engine import StreamEngine  # noqa: E402
from microwakeword_b200.playback import PlaybackGuard  # noqa: E402

HISTORY, ROWS, N_SAMPLES, MAX_DELAY = 48000, 4096, 24000, 16000


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "%s (nvidia-smi unavailable)" % torch.cuda.get_device_name(0)


def event_time(fn, calls):
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
    ap.add_argument("--calls", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("playback_guard_time.py measures the GPU kernels and needs a CUDA device; none is available")
    S, dev = a.streams, torch.device("cuda", 0)
    print("card: %s; %d streams, fp32 okay_nabu, history %d samples, %d rows of 10 s, L_ref %d" % (card(), S, HISTORY, ROWS,
                                                                                              N_SAMPLES + MAX_DELAY))
    clocks = ClockSampler(0)
    times = {}
    try:
        eng = StreamEngine(model_blob("f32"), n_streams=S)
        eng.set_audio_history(HISTORY)
        P = 1021
        audio = synth_audio_device(torch, P, HISTORY, 3, dev)[torch.arange(S, device=dev) % P].contiguous()
        probs = torch.empty((S, 1), dtype=torch.float32, device=dev)
        for i in range(HISTORY // 480):
            eng.step(audio[:, 480 * i:480 * (i + 1)].contiguous(), out=probs)
        chunk = audio[:, :480].contiguous()
        step = lambda: eng.step(chunk, out=probs)                                  # noqa: E731
        step()
        times["step() 480 samples"] = [event_time(step, 50) for _ in range(a.rounds)]
        pb = PlaybackGuard(model_blob("f32"), eng, slots=1024, rows=ROWS, capacity_s=10.0, n_samples=N_SAMPLES, max_delay=MAX_DELAY)
        gen = np.random.default_rng(0)
        playing = np.sort(gen.choice(S, ROWS, replace=False)).astype(np.int32)
        reply = audio[torch.from_numpy(playing).to(dev) % P, :HISTORY].contiguous()
        pb.play(playing, reply, starts=np.full(ROWS, eng.audio_samples_seen - HISTORY, np.int64))
        part = reply[:, :480].contiguous()
        heads = pb.heads()[1][playing]
        k = [0]

        def write():                                       # each call appends 480 samples at every row's head
            pb.play(playing, part, starts=heads + 480 * k[0])
            k[0] += 1
        write()
        times["play: %d rows x 480 samples" % ROWS] = [event_time(write, a.calls) for _ in range(a.rounds)]
        end = eng.audio_samples_seen
        for n in (32, 1024):
            ids = torch.from_numpy(gen.choice(playing, n, replace=False).astype(np.int32)).to(dev)
            ends = torch.full((n,), end, dtype=torch.int64, device=dev)
            fn = (lambda ids=ids, ends=ends: pb.check(ids, ends=ends))
            fn()
            before = pb.launch_count
            fn()
            per_call = pb.launch_count - before
            times["check: %d events, L_ref %d" % (n, N_SAMPLES + MAX_DELAY)] = [event_time(fn, a.calls) for _ in range(a.rounds)]
            scores = fn()[0].cpu().numpy()
            print("check of %d events: %d launches per call, %d heard" % (n, per_call, int((~np.isnan(scores)).sum())))
    finally:
        sampled = clocks.stop()
    print("SM clock during the run: median %s MHz (max %s MHz), throttle reasons seen: %s" %
          (sampled["sm_mhz"], sampled["sm_max_mhz"], ", ".join(sampled["reasons"]) or "none"))
    for key, t in times.items():
        print("%-58s best %8.3f ms per call (rounds %s)" % (key, min(t), " / ".join("%.3f" % x for x in t)))


if __name__ == "__main__":
    main()
