"""What per-stream input rates (mww_set_stream_rates) cost: 65 536 streams, fp32 okay_nabu.
  (a) every stream at 48 kHz: one handle with per-stream rates against one handle at 48 kHz -- the price of the gathered
      launch and the per-rate planning;
  (b) a quarter of the streams each at 8, 16, 44.1 and 48 kHz: one handle with per-stream rates against four handles of
      16 384 streams, one per rate, called one after the other.
Each for a 3 s device clip (n16 = 48 000) and a 30 ms live call (n16 = 480).  The arms alternate: each round runs every arm
`calls` times, two rounds.  Times are host wall clock around calls that end in a synchronise.  A separate torch.profiler
pass gives the resampler launches' own time per call (every resample_kernel instantiation).  Prints the card, its power
limit and the SM clock sampled during the timed rounds.
    python tools/stream_rates_time.py [calls] [live_calls]"""
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import ClockSampler, model_blob  # noqa: E402
from microwakeword_b200.engine import StreamEngine, inputs_for_rates  # noqa: E402

calls = int(sys.argv[1]) if len(sys.argv) > 1 else 3
live_calls = int(sys.argv[2]) if len(sys.argv) > 2 else 40
S = int(os.environ.get("STREAM_RATES_STREAMS", "65536"))
ROUNDS = 2
CLIP16, LIVE16 = 48000, 480


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "%s (nvidia-smi unavailable)" % torch.cuda.get_device_name(0)


def audio(rows, width, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randint(-12000, 12000, (rows, max(int(width), 1)), dtype=torch.int16, device="cuda", generator=g)


def scenario(title, blob, rates):
    """one per-stream-rate handle against one single-rate handle per rate over that rate's streams"""
    rates = np.asarray(rates, np.int32)
    per = StreamEngine(blob, S, 0, stream_rates=rates)
    groups = {int(r): int((rates == r).sum()) for r in np.unique(rates)}
    single = {r: StreamEngine(blob, n, 0, input_rate=r) for r, n in groups.items()}
    arms = {}
    for kind, n16, seed in (("3 s device clip", CLIP16, 31), ("30 ms live call", LIVE16, 32)):
        x = audio(S, inputs_for_rates(rates, 0, n16).max(), seed)
        xs = {r: audio(n, inputs_for_rates([r], 0, n16)[0], seed + r) for r, n in groups.items()}
        # every call below starts at a counter that is a multiple of n16, so D_s is the same in every call of a kind
        arms[(kind, "per-stream handle")] = (lambda x=x, n16=n16: per.predict_clip(x, samples16=n16))
        arms[(kind, "%d single-rate handle%s" % (len(single), "s" if len(single) > 1 else ""))] = (
            lambda xs=xs: [single[r].predict_clip(xs[r]) for r in single])
    for fn in arms.values():                                # warm-up
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    clocks = ClockSampler(0)
    for _ in range(ROUNDS):
        for k, fn in arms.items():
            n = calls if k[0].startswith("3 s") else live_calls
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(n):
                fn()
            torch.cuda.synchronize()
            times[k].append((time.perf_counter() - t0) * 1e3 / n)
    clk = clocks.stop()
    print("%s -- SM clock during the rounds: %s MHz, throttle reasons: %s" % (title, clk.get("sm_mhz"), clk.get("reasons")))
    for k, ts in times.items():
        print("  %-16s %-26s ms per call: %s" % (k[0], k[1], " / ".join("%.2f" % t for t in ts)))
    from torch.profiler import ProfilerActivity, profile
    for k, fn in arms.items():
        reps = 3 if k[0].startswith("3 s") else 20
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                fn()
            torch.cuda.synchronize()
        us = sum(e.device_time_total for e in prof.key_averages() if "resample_kernel" in e.key)
        print("  %-16s %-26s resampler launches: %.3f ms per call" % (k[0], k[1], us / 1e3 / reps))
    del per, single, arms
    torch.cuda.empty_cache()


def main():
    if not torch.cuda.is_available():
        raise SystemExit("stream_rates_time.py needs a CUDA device")
    print("card:", card())
    print("%d streams, fp32 okay_nabu" % S)
    blob = model_blob("f32")
    scenario("(a) every stream at 48 kHz", blob, np.full(S, 48000, np.int32))
    quarter = np.array([8000, 16000, 44100, 48000], np.int32)
    scenario("(b) a quarter each at 8, 16, 44.1 and 48 kHz", blob, quarter[np.arange(S) * 4 // S])


if __name__ == "__main__":
    main()
