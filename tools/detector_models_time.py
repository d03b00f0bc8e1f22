"""What gated multi-model detection costs a live loop (MultiModelDetector, mww_multi_detector_create): 65 536 streams, a
MultiModelEngine of two wake words and a VAD (fp32 okay_nabu, int8 okay_nabu, and fp32 okay_nabu as the VAD; all stride 3),
30 ms calls.

Loops, alternating inside each round (ms per call, host wall clock around work that ends in a synchronise):
  step only ........... eng.step(chunk)
  K plain detectors ... eng.step(chunk), one StreamDetector update per model (no gating possible), drains every 33 calls
  one gated update .... eng.step(chunk), det.update(probs) of one MultiModelDetector, det.drain() every 33 calls
  host gating ......... eng.step(chunk), every probability copied to pinned host memory, the gated rule in NumPy

Then the update kernels alone, device time from torch.profiler, at 1, 8 and 100 steps per call: detector_models_update_kernel
against the K detector_update_kernel launches it replaces, with the bytes a call moves computed from the shapes (each row's
state read and written, its probabilities read) beside the H100 SXM data sheet's 3.35 TB/s of HBM bandwidth.  Prints the
card, its power limit and the SM clock sampled during the timed rounds.  There is no CPU path: without a GPU it fails.
    python tools/detector_models_time.py [--streams 65536] [--calls 66] [--rounds 2]"""
import argparse
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import ClockSampler, model_blob, synth_audio_device  # noqa: E402

HBM_DATA_SHEET_GBS = 3350.0
WINDOWS, COOLDOWN, VAD, DRAIN_EVERY = [5, 5, 10], 25, 2, 33


def card():
    import subprocess
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "%s (nvidia-smi unavailable)" % torch.cuda.get_device_name(0)


class HostGated:
    """the gated rule on the host, all streams at once, for models that step together (one step each per 30 ms call): what
    a caller without the device detector runs after every step"""

    def __init__(self, S, cutoffs):
        self.hist = [np.zeros((w - 1, S), np.float32) for w in WINDOWS]
        self.seen = 0
        self.flag = [np.full(S, COOLDOWN, np.int32), np.full(S, COOLDOWN, np.int32), np.zeros(S, bool)]
        self.cutoffs = cutoffs

    def _push(self, k, p):
        h, w = self.hist[k], WINDOWS[k]
        s = h[0].copy()
        for j in range(1, w - 1):
            s += h[j]
        s += p
        h[:-1] = h[1:]
        h[-1] = p
        return s / np.float32(w)

    def update(self, probs):
        self.seen += 1
        avg = self._push(VAD, probs[VAD])
        active = self.flag[VAD] = (self.seen >= WINDOWS[VAD]) & (avg.astype(np.float64) > self.cutoffs[VAD])
        fired = 0
        for k in (0, 1):
            avg = self._push(k, probs[k])
            if self.seen < WINDOWS[k]:
                continue
            cd = self.flag[k]
            np.maximum(cd - 1, 0, out=cd)
            fire = (cd == 0) & (avg.astype(np.float64) > self.cutoffs[k]) & active
            cd[fire] = COOLDOWN
            fired += int(np.count_nonzero(fire))
        return fired


def update_bytes(S, n_steps):
    """bytes one call moves over every model: history, counter (8) and cooldown / flag (4) read and written, probabilities read"""
    return sum(S * (8 * (w - 1) + 24 + 4 * n_steps) for w in WINDOWS)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=65536)
    ap.add_argument("--calls", type=int, default=66)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("detector_models_time.py needs a CUDA device: the detector has no CPU path")
    from microwakeword_b200.detection import MultiModelDetector, StreamDetector
    from microwakeword_b200.engine import MultiModelEngine
    S = args.streams
    dev = torch.device("cuda", 0)
    eng = MultiModelEngine([model_blob("f32"), model_blob("int8"), model_blob("f32")], S, 0)
    assert eng.stride == [3, 3, 3]
    chunks = [synth_audio_device(torch, S, 480, 31 + i, dev) for i in range(4)]

    # wake cutoffs that about 1 % of the streams' best averages over 40 calls exceed; the VAD's at the median average
    for i in range(60):
        eng.step(chunks[i % 4])
    got = [[], [], []]
    for i in range(40):
        for k, p in enumerate(eng.step(chunks[i % 4])):
            got[k].append(p)
    cutoffs = []
    for k in range(3):
        avg = torch.cat(got[k], 1).unfold(1, WINDOWS[k], 1).mean(-1)
        cutoffs.append(float((avg.flatten()[::7].median() if k == VAD else torch.quantile(avg.max(1).values, 0.99)).item()))
    del got

    det = MultiModelDetector(eng, cutoffs, WINDOWS, COOLDOWN, vad=VAD)
    plain = [StreamDetector(S, cutoffs[k], WINDOWS[k], COOLDOWN) for k in range(3)]
    host = HostGated(S, cutoffs)
    pinned = [torch.empty((S, 1), dtype=torch.float32, pin_memory=True) for _ in range(3)]
    found = {"K plain detectors": 0, "one gated update": 0, "host gating": 0}

    def step_only(i):
        eng.step(chunks[i % 4])

    def k_plain(i):
        for d, p in zip(plain, eng.step(chunks[i % 4])):
            d.update(p)
        if (i + 1) % DRAIN_EVERY == 0:
            for k, d in enumerate(plain):
                ev, dropped = d.drain()
                if k != VAD:
                    found["K plain detectors"] += ev.size + dropped

    def gated(i):
        det.update(eng.step(chunks[i % 4]))
        if (i + 1) % DRAIN_EVERY == 0:
            ev, dropped = det.drain()
            found["one gated update"] += ev.size + dropped

    def host_gating(i):
        probs = eng.step(chunks[i % 4])
        if probs[0].shape[1]:
            for dst, p in zip(pinned, probs):
                dst.copy_(p, non_blocking=True)
            torch.cuda.synchronize()
            found["host gating"] += host.update([p.numpy()[:, 0] for p in pinned])

    arms = {"step only": step_only, "K plain detectors": k_plain, "one gated update": gated, "host gating": host_gating}
    for fn in arms.values():                               # warm-up of every arm
        for i in range(6):
            fn(i)
    for d in plain + [det]:
        d.drain()
    for k in found:
        found[k] = 0
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
    print("%d streams, models fp32 / int8 okay_nabu (wake) + fp32 okay_nabu (VAD), 30 ms calls, windows %s, cooldown %d, cutoffs %s;"
          % (S, WINDOWS, COOLDOWN, ", ".join("%.4f" % c for c in cutoffs)))
    print("ms per call, one figure per round (each detector arm sees only its own calls, so their detection counts differ):")
    for name in arms:
        print("  %-19s %s%s" % (name + ":", " / ".join("%.3f" % t for t in times[name]),
                                "   (%d wake detections)" % found[name] if name in found else ""))

    # the update kernels alone
    from torch.profiler import ProfilerActivity, profile
    print("update kernels alone (device time from torch.profiler, sum over a call's launches; bytes = state read and written")
    print("+ probabilities read, all three models; data sheet HBM %.0f GB/s).  Probabilities uniform in [0, 1.05 cutoff]:" % HBM_DATA_SHEET_GBS)
    del chunks
    g = torch.Generator(device=dev)
    g.manual_seed(5)
    for n_steps in (1, 8, 100):
        probs = [torch.rand((S, n_steps), generator=g, device=dev) * (1.05 * c) for c in cutoffs]
        reps = 100 if n_steps < 100 else 20
        res = {}
        for label, fn, key in (("one gated update", lambda: det.update(probs), "detector_models_update_kernel"),
                               ("K plain updates", lambda: [d.update(p) for d, p in zip(plain, probs)], "detector_update_kernel")):
            for _ in range(5):
                fn()
            per_round = []
            for _ in range(args.rounds):
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(reps):
                        fn()
                    torch.cuda.synchronize()
                per_round.append(sum(e.device_time_total for e in prof.key_averages() if key in e.key) / reps)
            for d in plain + [det]:
                d.drain()
            res[label] = per_round
        nbytes = update_bytes(S, n_steps)
        for label, per_round in res.items():
            us = min(per_round)
            print("  %6d streams x %3d steps, %-16s %s us per call, %d bytes, %.0f GB/s = %.0f %% of the data-sheet HBM rate"
                  % (S, n_steps, label + ":", " / ".join("%.1f" % t for t in per_round), nbytes, nbytes / us / 1e3,
                     100 * nbytes / us / 1e3 / HBM_DATA_SHEET_GBS))
        del probs


if __name__ == "__main__":
    main()
