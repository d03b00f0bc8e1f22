"""What moving streams between handles costs: fp32 okay_nabu, 65 536 streams per handle, rings rotated by live calls.
  (a) export_streams into records, import_streams into a second handle, for n = 1, 1 024 and all streams (timed apart);
  (b) the yardstick: the same record bytes copied device to device with torch.Tensor.copy_ (one copy; an export or an import
      each move that many bytes once);
  (c) what had to be done before: state_dict() on the source and load_state_dict() on the destination -- every stream of
      the handle through host memory, whatever n is; once per round, host wall clock;
  (d) copy_nn_state for n = 1 and 16: NN rings only (no window carry, noise estimates or pending rows), so not the same
      job; the first call after a live step also canonicalises the rings of both whole handles, and is reported apart.
The arms alternate over three rounds, every shape is warmed first, (a), (b) and (d) are timed with CUDA events around many
repetitions.  Rates are achieved copy rates: record bytes / time.  Ends by checking that after an import of every stream the
destination's next live call is bit-identical to the source's.  Prints the card, its power limit and the SM clock sampled
during the run.  There is no CPU path: without a CUDA device the script fails.
    python tools/stream_records_time.py [--streams 65536] [--rounds 3]"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import ClockSampler, model_blob, synth_audio_device  # noqa: E402
from microwakeword_b200.engine import StreamEngine  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--streams", type=int, default=65536)
ap.add_argument("--rounds", type=int, default=3)
args = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("stream_records_time.py needs a CUDA device: the record kernels have no CPU path")
S, ROUNDS = args.streams, max(args.rounds, 3)
dev = torch.device("cuda", 0)


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "%s (nvidia-smi unavailable)" % torch.cuda.get_device_name(0)


def event_ms(fn, reps):
    """ms per call of fn, CUDA events around `reps` calls"""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def serve(eng, live_calls, seed):
    """an 800-sample call (3 rows: no pending rows, 320 samples buffered), then 480-sample live calls that rotate the rings"""
    eng.predict_clip(synth_audio_device(torch, S, 800, seed, dev))
    for i in range(live_calls):
        eng.step(synth_audio_device(torch, S, 480, seed + 1 + i, dev))


def main():
    src, dst = StreamEngine(model_blob("f32"), n_streams=S, device=0), StreamEngine(model_blob("f32"), n_streams=S, device=0)
    serve(src, 5, 100)
    serve(dst, 9, 200)                     # same counters, another rotation
    record_bytes = int(src.stream_layout().record_bytes)
    rng = np.random.default_rng(0)
    shapes = [(n, rng.permutation(S)[:n].astype(np.int32), rng.permutation(S)[:n].astype(np.int32), reps)
              for n, reps in ((1, 200), (min(1024, S), 100), (S, 10))]
    times = {}

    def add(key, v):
        times.setdefault(key, []).append(v)

    recs = {n: src.export_streams(ids) for n, ids, _, _ in shapes}             # warm-up of every shape, and the import's input
    for n, ids, to, _ in shapes:
        dst.import_streams(to, recs[n])
        torch.empty_like(recs[n].data).copy_(recs[n].data)
    for e in (src, dst):
        e.step(synth_audio_device(torch, S, 480, 300, dev))
    dst.copy_nn_state([0], src, [0])
    torch.cuda.synchronize()

    for r in range(ROUNDS):
        for e in (src, dst):                         # arms (c) and (d) leave canonical rings behind: rotate them again
            e.step(synth_audio_device(torch, S, 480, 350 + r, dev))
        for n, ids, to, reps in shapes:
            add(("a_export", n), event_ms(lambda: src.export_streams(ids), reps))
            rec = recs[n]
            add(("a_import", n), event_ms(lambda: dst.import_streams(to, rec), reps))
            buf = torch.empty_like(rec.data)
            add(("b_copy_", n), event_ms(lambda: buf.copy_(rec.data), reps))
            del buf
        t0 = time.perf_counter()
        dst.load_state_dict(src.state_dict())
        torch.cuda.synchronize()
        add(("c_state_dict", S), (time.perf_counter() - t0) * 1e3)
        for n in (1, 16):
            ids = np.arange(n, dtype=np.int32)
            for e in (src, dst):                     # a live step in between: the rings are rotated again
                e.step(synth_audio_device(torch, S, 480, 400 + r, dev))
            add(("d_copy_nn_state_first", n), event_ms(lambda: dst.copy_nn_state(ids, src, ids), 1))
            add(("d_copy_nn_state_again", n), event_ms(lambda: dst.copy_nn_state(ids, src, ids), 100))

    # the check: every stream of src into dst (other ids, other audio so far; the same rotation, which the fp32 live kernel's
    # summation order depends on), then the same live audio to both
    serve(src, 3, 500)
    serve(dst, 3, 600)
    perm = rng.permutation(S).astype(np.int32)
    dst.import_streams(perm, src.export_streams(np.arange(S, dtype=np.int32)))
    audio = synth_audio_device(torch, S, 480, 700, dev)
    want = src.step(audio).cpu().numpy()
    moved = torch.empty_like(audio)
    moved[torch.from_numpy(perm.astype(np.int64)).to(dev)] = audio
    got = dst.step(moved).cpu().numpy()
    assert np.array_equal(got[perm].view(np.int32), want.view(np.int32)), "moved streams do not continue bit for bit"
    return record_bytes, times


print("card: %s; fp32 okay_nabu, %d streams per handle" % (card(), S))
clocks = ClockSampler(0)           # an nvidia-smi poller: stopped however the measurement ends
try:
    record_bytes, times = main()
finally:
    sampled = clocks.stop()
print("SM clock during the run: median %s MHz (max %s MHz), throttle reasons seen: %s" %
      (sampled["sm_mhz"], sampled["sm_max_mhz"], ", ".join(sampled["reasons"]) or "none"))
print("record: %d bytes per stream" % record_bytes)
for (arm, n), ms in times.items():
    line = "%-22s n = %-6d %s ms (rounds)" % (arm, n, " / ".join("%.4f" % t for t in ms))
    if arm[0] in "ab":
        line += "; %.1f MB, achieved copy rate %.1f GB/s (best round)" % (n * record_bytes / 1e6, n * record_bytes / min(ms) / 1e6)
    print(line)
print("check: after importing all %d streams the destination's next live call is bit-identical to the source's" % S)
