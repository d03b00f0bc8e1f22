"""What the input-rate resampler costs (mww_set_input_rate): 65 536 streams, fp32 okay_nabu, at 16 kHz (no resampler), 44.1
and 48 kHz, for a 3 s device clip, a 3 s host clip (pinned int16) and a 30 ms live call.  The arms alternate: each round runs
every rate's call `calls` times, two rounds.  Times are host wall clock around calls that end in a synchronise.  A separate
torch.profiler pass over device clips gives resample_kernel's own time, and its achieved rate from the bytes it must move
(input samples read + 16 kHz samples written, 2 bytes each).  Prints the card, its power limit and the SM clock sampled
during the timed rounds.
    python tools/resample_time.py [calls] [live_calls]"""
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import ClockSampler, model_blob, synth_audio_device  # noqa: E402
from microwakeword_b200.engine import StreamEngine, host_array  # noqa: E402

calls = int(sys.argv[1]) if len(sys.argv) > 1 else 3
live_calls = int(sys.argv[2]) if len(sys.argv) > 2 else 40
S = int(os.environ.get("RESAMPLE_STREAMS", "65536"))
RATES = (16000, 44100, 48000)
ROUNDS = 2


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "%s (nvidia-smi unavailable)" % torch.cuda.get_device_name(0)


def main():
    dev = torch.device("cuda", 0)
    blob = model_blob("f32")
    clip = {r: synth_audio_device(torch, S, 3 * r, 21, dev) for r in RATES}
    live = {r: synth_audio_device(torch, S, 3 * r // 100, 22, dev) for r in RATES}
    host = {}
    for r in RATES:
        host[r] = host_array((S, 3 * r), np.int16)
        host[r][:] = clip[r].cpu().numpy()
    eng = {r: StreamEngine(blob, S, 0, input_rate=r) for r in RATES}        # one engine per rate: every arm of a rate shares it
    arms = {
        "device 3 s clip": lambda r: eng[r].predict_clip(clip[r]),
        "host 3 s clip": lambda r: eng[r].predict_clip_host(host[r]),
        "live 30 ms call": lambda r: eng[r].step(live[r]),
    }
    n_calls = {"device 3 s clip": calls, "host 3 s clip": calls, "live 30 ms call": live_calls}
    for name, fn in arms.items():                       # warm-up
        for r in RATES:
            for _ in range(3):
                fn(r)
    torch.cuda.synchronize()
    times = {(name, r): [] for name in arms for r in RATES}
    clocks = ClockSampler(0)
    for _ in range(ROUNDS):
        for name, fn in arms.items():
            for r in RATES:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(n_calls[name]):
                    fn(r)
                torch.cuda.synchronize()
                times[(name, r)].append((time.perf_counter() - t0) * 1e3 / n_calls[name])
    clk = clocks.stop()
    print("card:", card(), "| SM clock during the rounds:", clk.get("sm_mhz"), "MHz, throttle reasons:", clk.get("reasons"))
    print("%d streams, fp32 okay_nabu; ms per call, one figure per round" % S)
    for name in arms:
        print("  %s: " % name + "   ".join("%d Hz %s" % (r, " / ".join("%.2f" % t for t in times[(name, r)])) for r in RATES))

    # the resampler kernel alone, from a profiled pass of device clips and live calls
    from torch.profiler import ProfilerActivity, profile
    for what, audio_of, reps in (("3 s device clip", clip, 3), ("30 ms live call", live, 20)):
        for r in RATES[1:]:
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(reps):
                    eng[r].predict_clip(audio_of[r])
                torch.cuda.synchronize()
            us = [e.device_time_total for e in prof.key_averages() if "resample_kernel" in e.key]
            n_in = audio_of[r].shape[1]
            n_out = (n_in * 16000 + r - 1) // r
            ms = sum(us) / 1e3 / reps
            gbs = S * (n_in + n_out) * 2 / (ms / 1e3) / 1e9 if ms > 0 else float("nan")
            print("  resample_kernel, %s at %d Hz: %.3f ms per call, %.0f GB/s (input read + 16 kHz written)" % (what, r, ms, gbs))


if __name__ == "__main__":
    main()
