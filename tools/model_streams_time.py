"""What per-model stream sets save: K = 4 models (fp32 and int8 okay_nabu containers, alternating) over one frontend at
65 536 streams, three MultiModelEngines fed the same audio:
  (a) every model on all streams,
  (b) each stream on one model, in contiguous blocks of S / 4 streams (rows read in place),
  (c) each stream on one model, interleaved: model k on streams s % 4 == k (rows gathered per tile),
for a 3 s clip from device memory (predict_clip), a 3 s clip from pinned host memory (predict_clip_host) and 480-sample
live calls (step).  The arms alternate, three rounds, each runs its calls `calls` times per round; ms per call is reported
per round.  The last call's probabilities of (b) and (c) are compared bit for bit with the member rows of (a).  Prints the
card, its power limit and SM clock read in the same run, and each arm's NN state bytes.
    python tools/model_streams_time.py [clip_calls] [live_calls]"""
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import model_blob, synth_audio_device  # noqa: E402
from microwakeword_b200.engine import MultiModelEngine, host_array  # noqa: E402

clip_calls = int(sys.argv[1]) if len(sys.argv) > 1 else 3
live_calls = int(sys.argv[2]) if len(sys.argv) > 2 else 100
S = int(os.environ.get("MODEL_STREAMS_STREAMS", "65536"))
K = 4
ROUNDS = 3
dev = torch.device("cuda", 0)


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "%s (nvidia-smi unavailable)" % torch.cuda.get_device_name(0)


def to_np(x):
    return x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)


print("card: %s; %d streams, %d models" % (card(), S, K))
blobs = [model_blob(k) for k in (["f32", "int8"] * K)[:K]]
q = S // K
arms = {"all": MultiModelEngine(blobs, S),
        "blocks": MultiModelEngine(blobs, S, streams=[np.arange(k * q, (k + 1) * q if k < K - 1 else S, dtype=np.int32) for k in range(K)]),
        "interleaved": MultiModelEngine(blobs, S, streams=[np.arange(k, S, K, dtype=np.int32) for k in range(K)])}
for name, e in arms.items():
    nn = sum(e.streams[k].size * e.state_elements[k] * (1 if e.is_quantized[k] else 4) for k in range(K))
    print("%-12s NN ring state %.2f GB" % (name, nn / 1e9))

d_clip = synth_audio_device(torch, S, 48000, 11, dev)
h_clip = host_array((S, 48000), np.int16, 0)
h_clip[:] = d_clip.cpu().numpy()
d_live = synth_audio_device(torch, S, 480, 12, dev)
cases = {"device clip 3 s": (lambda e: e.predict_clip(d_clip), clip_calls),
         "host clip 3 s": (lambda e: e.predict_clip_host(h_clip), clip_calls),
         "live 480": (lambda e: e.step(d_live), live_calls)}
for case, (fn, calls) in cases.items():
    for e in arms.values():                                   # warm-up: modules, scratch, staging buffers
        fn(e)
    torch.cuda.synchronize()
    times, last = {a: [] for a in arms}, {}
    for _ in range(ROUNDS):
        for a, e in arms.items():
            t0 = time.perf_counter()
            for _ in range(calls):
                last[a] = fn(e)
            torch.cuda.synchronize()
            times[a].append((time.perf_counter() - t0) * 1e3 / calls)
    for a in ("blocks", "interleaved"):                       # every arm saw the same calls: member rows agree bit for bit
        for k in range(K):
            g, w = to_np(last[a][k]), to_np(last["all"][k])[arms[a].streams[k]]
            assert g.shape == w.shape and np.array_equal(g.view(np.int32), w.view(np.int32)), (case, a, k)
    med = {a: float(np.median(t)) for a, t in times.items()}
    print("%-16s " % case + "   ".join("%s %s ms" % (a, " / ".join("%.2f" % t for t in times[a])) for a in arms) +
          "   (ms per call, rounds; median all / blocks %.2f, all / interleaved %.2f)" % (med["all"] / med["blocks"], med["all"] / med["interleaved"]))
print("member rows of (b) and (c) equal (a) bit for bit in every case")
print("card after: %s" % card())
