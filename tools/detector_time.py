"""What detection costs a live loop (StreamDetector, mww_detector_*): 65 536 streams, fp32 okay_nabu, 30 ms calls.

Loops, alternating inside each round (ms per call, host wall clock around work that ends in a synchronise):
  step only .......... eng.step(chunk)
  host detection ..... eng.step(chunk), every probability copied to a pinned host buffer, the same rule in NumPy over all rows
  device detection ... eng.step(chunk), det.update(probs), det.drain() every 33 calls

Then detector_update_kernel alone, its device time from torch.profiler over many launches, at 1 step per row (the live shape, thread per row),
on either side of the step count where the launcher changes form, and at 100 steps (a 3 s clip, warp per row), with the
bytes a call has to move computed from the shapes -- the row's state read and written, its probabilities read -- and the
rate that gives, beside the H100 SXM data sheet's 3.35 TB/s of HBM bandwidth: the bound of a kernel that only moves bytes.
Prints the card, its power limit and the SM clock sampled during the timed rounds.  There is no CPU path: without a GPU it fails.
    python tools/detector_time.py [--rows 65536] [--calls 66] [--rounds 2]"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import ClockSampler, model_blob, synth_audio_device  # noqa: E402
from microwakeword_b200.detection import StreamDetector  # noqa: E402
from microwakeword_b200.engine import StreamEngine  # noqa: E402

HBM_DATA_SHEET_GBS = 3350.0
WINDOW, COOLDOWN, DRAIN_EVERY = 5, 25, 33


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "%s (nvidia-smi unavailable)" % torch.cuda.get_device_name(0)


class HostDetector:
    """the rule on the host, all rows at once: what a caller without the device detector runs after every step"""

    def __init__(self, n_rows, cutoff):
        self.hist = np.zeros((WINDOW - 1, n_rows), np.float32)
        self.seen = 0
        self.cooldown = np.full(n_rows, COOLDOWN, np.int32)
        self.cutoff = cutoff

    def update(self, p):
        s = self.hist[0].copy()
        for j in range(1, WINDOW - 1):
            s += self.hist[j]
        s += p
        self.hist[:-1] = self.hist[1:]
        self.hist[-1] = p
        self.seen += 1
        if self.seen < WINDOW:
            return np.zeros(0, np.int64)
        avg = s / np.float32(WINDOW)
        np.maximum(self.cooldown - 1, 0, out=self.cooldown)
        fire = (self.cooldown == 0) & (avg.astype(np.float64) > self.cutoff)
        self.cooldown[fire] = COOLDOWN
        return np.nonzero(fire)[0]


def update_bytes(n_rows, n_steps, window):
    """bytes one update call must move: history, counter (8) and cooldown (4) read and written, the probabilities read"""
    return n_rows * (8 * (window - 1) + 24 + 4 * n_steps)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=65536)
    ap.add_argument("--calls", type=int, default=66)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--steps", default="", help="steps per row of the kernel-alone part (default: 1, either side of the form change, 100)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("detector_time.py needs a CUDA device: the detector has no CPU path")
    S = args.rows
    dev = torch.device("cuda", 0)
    eng = StreamEngine(model_blob("f32"), S, 0)
    chunks = [synth_audio_device(torch, S, 480, 31 + i, dev) for i in range(4)]

    # a cutoff inside the range the model produces on this audio once the streams have run for a while: over 40 calls the
    # best moving average of about 1 % of the streams exceeds it
    for i in range(60):
        eng.step(chunks[i % 4])
    probe = torch.cat([eng.step(chunks[i % 4]) for i in range(40)], 1)
    cutoff = float(torch.quantile(probe.unfold(1, WINDOW, 1).mean(-1).max(1).values, 0.99))

    det = StreamDetector(S, cutoff, WINDOW, COOLDOWN)
    host_det = HostDetector(S, cutoff)
    pinned = torch.empty((S, 1), dtype=torch.float32, pin_memory=True)
    found = {"host detection": 0, "device detection": 0}

    def step_only(i):
        eng.step(chunks[i % 4])

    def host_detection(i):
        p = eng.step(chunks[i % 4])
        if p.shape[1]:
            pinned.copy_(p, non_blocking=True)
            torch.cuda.synchronize()
            found["host detection"] += host_det.update(pinned.numpy()[:, 0]).size

    def device_detection(i):
        det.update(eng.step(chunks[i % 4]))
        if (i + 1) % DRAIN_EVERY == 0:
            ev, dropped = det.drain()
            found["device detection"] += ev.size + dropped

    arms = {"step only": step_only, "host detection": host_detection, "device detection": device_detection}
    for fn in arms.values():                              # warm-up of every arm
        for i in range(6):
            fn(i)
    torch.cuda.synchronize()
    det.drain()
    times = {name: [] for name in arms}
    clocks = ClockSampler(0)
    for _ in range(args.rounds):
        for name, fn in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for i in range(args.calls):
                fn(i)
            torch.cuda.synchronize()
            times[name].append((time.perf_counter() - t0) * 1e3 / args.calls)
    clk = clocks.stop()
    print("card:", card(), "| SM clock during the rounds:", clk.get("sm_mhz"), "MHz, throttle reasons:", clk.get("reasons"))
    print("%d streams, fp32 okay_nabu, 30 ms calls, window %d, cooldown %d, cutoff %.4f; ms per call, one figure per round" % (S, WINDOW, COOLDOWN, cutoff))
    for name in arms:
        print("  %-17s %s%s" % (name + ":", " / ".join("%.3f" % t for t in times[name]),
                                "   (%.1f detections per call)" % (found[name] / (args.calls * args.rounds + 6)) if name in found else ""))
    print("  probabilities leaving the GPU per call: host detection %d bytes, device detection %d bytes of events per drain at most"
          % (S * 4, det.capacity * 24))

    # the update kernel alone
    from microwakeword_b200 import _lib
    warp_min = int(open(os.path.join(os.path.dirname(_lib.SO_PATH), "csrc", "mww_detector.h")).read().split("kDetectorWarpMinSteps = ")[1].split(";")[0])
    from torch.profiler import ProfilerActivity, profile
    step_list = [int(v) for v in args.steps.split(",")] if args.steps else [1, warp_min - 1, warp_min, 100]
    print("detector_update_kernel alone (kernel time from torch.profiler; bytes = state read and written + probabilities read;")
    print("data sheet HBM %.0f GB/s).  At %d rows the state and one step's probabilities stay in the 50 MB L2 between back-to-back calls," % (HBM_DATA_SHEET_GBS, S))
    print("which a live loop's step kernels would evict; %d rows do not fit, so those calls read and write HBM.  Probabilities are uniform" % (64 * S))
    print("in [0, 1.05 cutoff] (few rows fire) or, `dense`, in [0, 2 cutoff] (every row fires as often as the cooldown allows):")
    del eng, chunks, probe
    for rows in (S, 64 * S):
        g = torch.Generator(device=dev)
        g.manual_seed(5)
        d = det if rows == S else StreamDetector(rows, cutoff, WINDOW, COOLDOWN)
        for n_steps, scale in [(n, 1.05) for n in step_list] + [(n, 2.0) for n in (1, 100) if n in step_list]:
            probs = torch.rand((rows, n_steps), generator=g, device=dev) * (scale * cutoff)
            reps = 100 if rows * n_steps < (1 << 24) else 20
            for _ in range(5):
                d.update(probs)
            d.drain()
            per_round, events = [], 0
            for _ in range(args.rounds):
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(reps):
                        d.update(probs)
                    torch.cuda.synchronize()
                per_round.append(sum(e.device_time_total for e in prof.key_averages() if "detector_update_kernel" in e.key) / reps)
                ev, dropped = d.drain()
                events = (ev.size + dropped) / reps
            nbytes = update_bytes(rows, n_steps, WINDOW)
            us = min(per_round)
            print("  %8d rows x %3d steps%s (%s per row, %.0f events per call): %s us per call, %d bytes, %.0f GB/s = %.0f %% of the data-sheet HBM rate"
                  % (rows, n_steps, " dense" if scale > 1.5 else "", "warp" if n_steps >= warp_min else "thread", events,
                     " / ".join("%.1f" % t for t in per_round), nbytes, nbytes / us / 1e3, 100 * nbytes / us / 1e3 / HBM_DATA_SHEET_GBS))
            del probs


if __name__ == "__main__":
    main()
