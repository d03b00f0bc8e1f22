"""What moving detector rows costs (mww_export_detector_rows / mww_import_detector_rows): packed device records against the
whole-detector state round trip through the host that was the only way before.

  plain ....... a 65 536-row StreamDetector (window 5, 48-byte records): export of 1, 1 024 and 65 536 rows, and their
                import into another 65 536-row detector at other indices
  gated ....... a MultiModelDetector with two wake words and a VAD over a 65 536-stream MultiModelEngine (fp32 and int8
                okay_nabu as the wake words, fp32 okay_nabu as the VAD, windows 5, 5 and 10): the same sizes
  state dict .. the same move done the old way: state_dict() of both detectors, the rows copied on the host,
                load_state_dict() on the destination (what moving any number of rows cost before)

Export and import are timed with CUDA events around --reps back-to-back Python calls each (host id list in, one launch,
records on the device), so the figure is a whole call: the host work between launches (id checks, the cutoff bookkeeping)
leaves the GPU idle and counts.  Beside it, torch.profiler gives the pack / unpack kernel's own device time.  The
state-dict path is timed with the host clock, as it synchronises the device itself.  The arms alternate inside each round and
the best round is printed.  Prints the card, its power limit and the SM clock sampled during the run.  There is no CPU
path: without a GPU it fails.
    python tools/detector_records_time.py [--rows 65536] [--rounds 3] [--reps 50]"""
import argparse
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import ClockSampler, model_blob  # noqa: E402

SIZES = (1, 1024, 65536)


def card():
    import subprocess
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "%s (nvidia-smi unavailable)" % torch.cuda.get_device_name(0)


def event_ms(fn, reps):
    """time per call of fn() on the device's timeline over reps calls, idle gaps between launches included"""
    fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def kernel_ms(fn, name, reps=5):
    """device time of the kernels whose name holds `name`, per call of fn(), from torch.profiler"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.key_averages() if name in e.key and (name != "pack_detector" or "unpack" not in e.key))
    return us / 1e3 / reps


def wall_ms(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3


def move_by_state(src, dst, src_ids, dst_ids, multi):
    s, d = src.state_dict(), dst.state_dict()
    if multi:
        for k, (a, b) in enumerate(zip(s["models"], d["models"])):
            if a is not None:
                for key in a:
                    b[key][dst_ids] = a[key][src_ids]
    else:
        for key in s:
            d[key][dst_ids] = s[key][src_ids]
    dst.load_state_dict(d)


def run_arms(name, src, dst, n_ids, multi, args, rng):
    export = src.export_streams if multi else src.export_rows
    imp = dst.import_streams if multi else dst.import_rows
    best = {}
    for _ in range(args.rounds):
        for n in SIZES:
            if n > n_ids:
                continue
            src_ids = rng.permutation(n_ids)[:n].astype(np.int32)
            dst_ids = rng.permutation(n_ids)[:n].astype(np.int32)
            rec = export(src_ids)
            arms = {"export": lambda: export(src_ids), "import": lambda: imp(dst_ids, rec),
                    "state_dict": lambda: move_by_state(src, dst, src_ids, dst_ids, multi)}
            for arm, fn in arms.items():
                ms = wall_ms(fn) if arm == "state_dict" else event_ms(fn, args.reps)
                key = (n, arm)
                best[key] = min(best.get(key, ms), ms)
            for arm, kernel in (("export", "pack_detector"), ("import", "unpack_detector")):
                ms = kernel_ms(arms[arm], kernel)
                key = (n, arm + " kernel")
                best[key] = min(best.get(key, ms), ms)
    rb = int(src.layout().record_bytes)
    print("%s: %d-byte records, %d ids" % (name, rb, n_ids))
    for n in SIZES:
        if (n, "export") not in best:
            continue
        print("  %6d rows  call: export %7.3f ms  import %7.3f ms | kernel: pack %7.3f ms  unpack %7.3f ms | "
              "state_dict round trip %8.2f ms  (%.2f MB of records)"
              % (n, best[(n, "export")], best[(n, "import")], best[(n, "export kernel")], best[(n, "import kernel")],
                 best[(n, "state_dict")], n * rb / 1e6))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=65536)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("detector_records_time.py needs a CUDA device: the detector has no CPU path")
    from microwakeword_b200.detection import MultiModelDetector, StreamDetector
    from microwakeword_b200.engine import MultiModelEngine
    R = args.rows
    rng = np.random.default_rng(0)
    clocks = ClockSampler(0)
    src, dst = StreamDetector(R, 0.7, 5, 25), StreamDetector(R, 0.7, 5, 25)
    probs = torch.from_numpy(rng.random((R, 40)).astype(np.float32)).cuda()
    src.update(probs)                                     # warm rows, some in cooldown
    run_arms("plain (StreamDetector, window 5)", src, dst, R, False, args, rng)
    del src, dst
    eng = MultiModelEngine([model_blob("f32"), model_blob("int8"), model_blob("f32")], R, 0)
    src = MultiModelDetector(eng, [0.9, 0.9, 0.5], windows=[5, 5, 10], cooldown_slices=25, vad=2)
    dst = MultiModelDetector(eng, [0.9, 0.9, 0.5], windows=[5, 5, 10], cooldown_slices=25, vad=2)
    run_arms("gated (MultiModelDetector, WAKE 5 + WAKE 5 + VAD 10)", src, dst, R, True, args, rng)
    c = clocks.stop()
    print("card: %s; SM clock median %s MHz (max %s), throttle reasons %s" % (card(), c["sm_mhz"], c["sm_max_mhz"], c["reasons"] or "none"))


if __name__ == "__main__":
    main()
