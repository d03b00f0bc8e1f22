"""What float32 HOST audio costs: a 3 s clip call and a 480-sample live call at 65 536 streams from host buffers, three ways --
  (a) int16 pinned audio -> predict_clip_host,
  (b) float32 pinned audio -> predict_clip_host (the floats cross PCIe and are converted inside the frontend kernels),
  (c) float32 pinned audio -> audio_utils.to_int16 on the host -> predict_clip_host of its (pageable) result: what
      Model.step did with float32 numpy before the float host path existed.
The arms alternate: each round runs every arm `calls` times, and there are two rounds.  Each arm has its own engine fed the
same audio, so their probabilities must be bit-identical (checked).  Times are host wall clock around the synchronous calls.
Also times to_int16 alone.  Prints the card, its power limit and the SM clock sampled during the run.
    python tools/float_host_time.py [f32|int8] [clip_calls] [live_calls]"""
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import ClockSampler, model_blob, synth_audio_device  # noqa: E402
from microwakeword_b200.audio.audio_utils import to_int16  # noqa: E402
from microwakeword_b200.engine import StreamEngine, host_array  # noqa: E402

kind = sys.argv[1] if len(sys.argv) > 1 else "f32"
clip_calls = int(sys.argv[2]) if len(sys.argv) > 2 else 3
live_calls = int(sys.argv[3]) if len(sys.argv) > 3 else 50
S = int(os.environ.get("FLOAT_HOST_STREAMS", "65536"))
ROUNDS = 2


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "%s (nvidia-smi unavailable)" % torch.cuda.get_device_name(0)


def measure(n_samples, calls):
    """-> {arm: [ms per call, one per round]}, to_int16 alone in ms per call"""
    i16 = host_array((S, n_samples), np.int16)
    i16[:] = synth_audio_device(torch, S, n_samples, 11, torch.device("cuda", 0)).cpu().numpy()
    f32 = host_array((S, n_samples), np.float32)
    np.multiply(i16, np.float32(1 / 32768), out=f32)      # exact; to_int16 gives back the same samples
    assert np.array_equal(to_int16(f32[:64]), i16[:64])

    arms = {"a_int16": lambda eng, out: eng.predict_clip_host(i16, out=out),
            "b_float32": lambda eng, out: eng.predict_clip_host(f32, out=out),
            "c_host_to_int16": lambda eng, out: eng.predict_clip_host(np.ascontiguousarray(to_int16(f32)), out=out)}
    engines = {k: StreamEngine(model_blob(kind), n_streams=S, device=0) for k in arms}
    outs = {k: host_array((S, 128), np.float32) for k in arms}
    last = {}
    for k, fn in arms.items():                           # warm-up: module load, staging buffers, steady buffered count
        for _ in range(2):
            last[k] = fn(engines[k], outs[k])
    times = {k: [] for k in arms}
    for _ in range(ROUNDS):
        for k, fn in arms.items():
            t0 = time.perf_counter()
            for _ in range(calls):
                last[k] = fn(engines[k], outs[k])
            times[k].append((time.perf_counter() - t0) * 1e3 / calls)
    ref = last["a_int16"].view(np.int32)
    for k in arms:
        assert last[k].shape == last["a_int16"].shape and np.array_equal(last[k].view(np.int32), ref), k
    t0 = time.perf_counter()
    for _ in range(calls):
        to_int16(f32)
    convert_ms = (time.perf_counter() - t0) * 1e3 / calls
    for e in engines.values():
        e.close()
    return times, convert_ms


print("card: %s; model %s, %d streams, pinned audio buffers" % (card(), kind, S))
results = []
clocks = ClockSampler(0)           # an nvidia-smi poller: stopped however the measurement ends (failed check, OOM, Ctrl-C)
try:
    for name, n, calls in (("clip 3 s", 48000, clip_calls), ("live 480", 480, live_calls)):
        results.append((name, n) + measure(n, calls))
finally:
    sampled = clocks.stop()
print("SM clock during the run: median %s MHz (max %s MHz), throttle reasons seen: %s" %
      (sampled["sm_mhz"], sampled["sm_max_mhz"], ", ".join(sampled["reasons"]) or "none"))
for name, n, times, convert_ms in results:
    for k in times:
        print("%-9s %-16s call %s ms (rounds)" % (name, k, " / ".join("%.2f" % t for t in times[k])))
    print("%-9s to_int16 alone   %.2f ms per call (%.1f MB of float32)" % (name, convert_ms, S * n * 4 / 1e6))
