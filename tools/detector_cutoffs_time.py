"""What per-row cutoffs cost (mww_set_detector_cutoffs, mww_set_multi_detector_cutoffs): the same detectors in uniform and in
per-row mode, alternating inside each round.

  plain kernel alone ... StreamDetector.update at --rows (65 536 and 4 194 304 by default) x 1, 8, 47, 48 and 100 steps
                         (47 is the thread form's last step count, 48 the warp form's first); device time from torch.profiler,
                         with the bytes a call moves computed from the shapes beside the H100 SXM data sheet's 3.35 TB/s
  models kernel alone .. MultiModelDetector.update over fp32 and int8 okay_nabu (wake) and fp32 okay_nabu (VAD) at 65 536
                         streams x 1, 8 and 100 steps
  live loop ............ StreamEngine.step of 30 ms + StreamDetector.update, 65 536 streams, host wall clock per call

Three arms alternate inside each round: uniform mode at cutoff 0.7; per-row mode with every row at 0.7, which fires exactly
the uniform arm's events and so isolates what the mode itself costs; and per-row mode with cutoffs drawn from three levels
(0.5, 0.7, 0.9) and random values, as a server would hold them, which fires other events than the first two (the live loop
runs the first two).  Prints the card, its power limit and the SM clock sampled during the run.  There is no CPU path:
without a GPU it fails.
    python tools/detector_cutoffs_time.py [--rows 65536,4194304] [--rounds 3] [--calls 66]"""
import argparse
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import ClockSampler, model_blob, synth_audio_device  # noqa: E402

HBM_DATA_SHEET_GBS = 3350.0
WINDOW, COOLDOWN, LEVELS = 5, 25, (0.5, 0.7, 0.9)


def card():
    import subprocess
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "%s (nvidia-smi unavailable)" % torch.cuda.get_device_name(0)


def row_cutoffs(n, seed=1):
    rng = np.random.default_rng(seed)
    c = np.asarray(LEVELS, np.float64)[rng.integers(0, 3, n)]
    rand = rng.random(n) < 0.1
    c[rand] = rng.uniform(0.4, 0.95, int(rand.sum()))
    return c


def plain_bytes(rows, n_steps, per_row):
    """history, counter (8) and cooldown (4) read and written, probabilities read, and the row's cutoff in per-row mode"""
    return rows * (8 * (WINDOW - 1) + 24 + 4 * n_steps + (8 if per_row else 0))


def kernel_us(fn, key, reps, rounds, drain):
    """device time per launch of the kernels whose name holds `key` (each call is one launch), one figure per round"""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(3):
        fn()
    drain()
    out = []
    for _ in range(rounds):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                fn()
            torch.cuda.synchronize()
        ev = [e for e in prof.key_averages() if key in e.key]
        n = sum(e.count for e in ev)
        if n:                                              # a round in which the profiler recorded no kernel is left out
            out.append(sum(e.device_time_total for e in ev) / n)
        drain()
    return out


ARMS = ("uniform", "per-row 0.7", "per-row mix")


def measure(args, lines):
    from microwakeword_b200.detection import MultiModelDetector, StreamDetector
    from microwakeword_b200.engine import MultiModelEngine, StreamEngine
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev)
    g.manual_seed(5)

    # the plain kernel alone
    for R in (int(r) for r in args.rows.split(",")):
        dets = {a: StreamDetector(R, LEVELS[1], WINDOW, COOLDOWN, capacity=1 << 20) for a in ARMS}
        dets["per-row 0.7"].set_cutoffs(np.arange(R), LEVELS[1])
        dets["per-row mix"].set_cutoffs(np.arange(R), row_cutoffs(R))
        for n_steps in (1, 8, 47, 48, 100):
            probs = torch.rand((R, n_steps), generator=g, device=dev)
            reps = max(3, min(200, int(2e8 // (R * (n_steps + 10)))))
            res = {a: [] for a in ARMS}
            for _ in range(args.rounds):                    # the arms alternate inside each round
                for label, det in dets.items():
                    res[label].extend(kernel_us(lambda: det.update(probs), "detector_update_kernel", reps, 1, det.drain))
            for label, per_round in res.items():
                us = min(per_round)
                nb = plain_bytes(R, n_steps, label != "uniform")
                lines.append("  plain  %8d rows x %3d steps, %-12s %s us, %.0f GB/s = %.0f %% of the data-sheet HBM rate"
                             % (R, n_steps, label + ":", " / ".join("%.1f" % t for t in per_round), nb / us / 1e3,
                                100 * nb / us / 1e3 / HBM_DATA_SHEET_GBS))
            u = min(res["uniform"])
            lines.append("  plain  %8d rows x %3d steps: per-row 0.7 / uniform = %.3f, per-row mix / uniform = %.3f"
                         % (R, n_steps, min(res["per-row 0.7"]) / u, min(res["per-row mix"]) / u))
            del probs
        del dets
        torch.cuda.empty_cache()

    # the models kernel alone
    S = 65536
    eng = MultiModelEngine([model_blob("f32"), model_blob("int8"), model_blob("f32")], S, 0)
    cut = [LEVELS[1], LEVELS[1], 0.5]
    dets = {a: MultiModelDetector(eng, cut, [5, 5, 10], COOLDOWN, vad=2, capacity=1 << 20) for a in ARMS}
    for k in range(3):
        dets["per-row 0.7"].set_cutoffs(k, np.arange(S), cut[k])
        dets["per-row mix"].set_cutoffs(k, np.arange(S), row_cutoffs(S, 10 + k) if k < 2 else 0.5)
    for n_steps in (1, 8, 100):
        probs = [torch.rand((S, n_steps), generator=g, device=dev) for _ in range(3)]
        res = {a: [] for a in ARMS}
        for _ in range(args.rounds):
            for label, det in dets.items():
                res[label].extend(kernel_us(lambda: det.update(probs), "detector_models_update_kernel",
                                            50 if n_steps < 100 else 10, 1, det.drain))
        for label, per_round in res.items():
            lines.append("  models %8d streams x %3d steps, %-12s %s us" % (S, n_steps, label + ":", " / ".join("%.1f" % t for t in per_round)))
        u = min(res["uniform"])
        lines.append("  models %8d streams x %3d steps: per-row 0.7 / uniform = %.3f, per-row mix / uniform = %.3f"
                     % (S, n_steps, min(res["per-row 0.7"]) / u, min(res["per-row mix"]) / u))
    del eng, dets
    torch.cuda.empty_cache()

    # a live loop
    eng = StreamEngine(model_blob("f32"), S, 0)
    chunks = [synth_audio_device(torch, S, 480, 31 + i, dev) for i in range(4)]
    dets = {a: StreamDetector(S, LEVELS[1], WINDOW, COOLDOWN) for a in ARMS[:2]}
    dets["per-row 0.7"].set_cutoffs(np.arange(S), LEVELS[1])
    times = {a: [] for a in dets}
    for i in range(10):
        for det in dets.values():
            det.update(eng.step(chunks[i % 4]))
    for _ in range(args.rounds):
        for label, det in dets.items():
            det.drain()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for i in range(args.calls):
                det.update(eng.step(chunks[i % 4]))
            torch.cuda.synchronize()
            times[label].append((time.perf_counter() - t0) * 1e3 / args.calls)
    for label, t in times.items():
        lines.append("  live loop, %d streams, 30 ms step() + update(), %-12s %s ms per call" % (S, label + ":", " / ".join("%.3f" % x for x in t)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", default="65536,4194304")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--calls", type=int, default=66)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("detector_cutoffs_time.py needs a CUDA device: the detector has no CPU path")
    lines = []
    clocks = ClockSampler(0)           # an nvidia-smi poller: stopped however the measurement ends (failed check, OOM, Ctrl-C)
    try:
        measure(args, lines)
    finally:
        clk = clocks.stop()
    print("card:", card(), "| SM clock during the run:", clk.get("sm_mhz"), "MHz, throttle reasons:", clk.get("reasons"))
    print("window %d, cooldown %d; uniform at %.1f; mix: %s and random values; device times from torch.profiler" % (WINDOW, COOLDOWN, LEVELS[1], LEVELS))
    print("\n".join(lines))


if __name__ == "__main__":
    main()
