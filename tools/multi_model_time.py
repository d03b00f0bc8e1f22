"""What several models over one frontend save: K = 1, 2, 4 models (fp32 and int8 okay_nabu containers, repeated) at 65 536
streams, one MultiModelEngine against K StreamEngines fed the same audio, for
  (a) a 3 s clip from device memory (predict_clip),
  (b) a 3 s clip from pinned host memory (predict_clip_host; the audio crosses PCIe once per engine),
  (c) 480-sample live calls (step).
The two arms alternate, three rounds, each runs its calls `calls` times per round; ms per call is reported per round.  The
last call's probabilities of every model are compared bit for bit between the arms.  Prints the card, its power limit and
SM clock read in the same run.
    python tools/multi_model_time.py [clip_calls] [live_calls]"""
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import model_blob, synth_audio_device  # noqa: E402
from microwakeword_b200.engine import MultiModelEngine, StreamEngine, host_array  # noqa: E402

clip_calls = int(sys.argv[1]) if len(sys.argv) > 1 else 3
live_calls = int(sys.argv[2]) if len(sys.argv) > 2 else 100
S = int(os.environ.get("MULTI_MODEL_STREAMS", "65536"))
ROUNDS = 3
dev = torch.device("cuda", 0)


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "%s (nvidia-smi unavailable)" % torch.cuda.get_device_name(0)


def measure(K, d_clip, h_clip, d_live):
    kinds = (["f32", "int8"] * K)[:K]
    blobs = [model_blob(k) for k in kinds]
    multi = MultiModelEngine(blobs, S)
    singles = [StreamEngine(b, S) for b in blobs]
    cases = {"device clip 3 s": (lambda e: e.predict_clip(d_clip), clip_calls, True),
             "host clip 3 s": (lambda e: e.predict_clip_host(h_clip), clip_calls, False),
             "live 480": (lambda e: e.step(d_live), live_calls, True)}
    res = {}
    for name, (fn, calls, on_device) in cases.items():
        arms = {"multi": lambda: fn(multi), "separate": lambda: [fn(e) for e in singles]}
        for run in arms.values():                         # warm-up: modules, scratch, staging buffers
            run()
        torch.cuda.synchronize()
        times, last = {a: [] for a in arms}, {}
        for _ in range(ROUNDS):
            for a, run in arms.items():
                t0 = time.perf_counter()
                for _ in range(calls):
                    last[a] = run()
                torch.cuda.synchronize()
                times[a].append((time.perf_counter() - t0) * 1e3 / calls)
        for k in range(K):                                # both arms saw the same calls: same state, same scores
            g, w = last["multi"][k], last["separate"][k]
            if on_device:
                assert torch.equal(g.contiguous().view(torch.int32), w.contiguous().view(torch.int32)), (name, k)
            else:
                assert np.array_equal(g.view(np.int32), w.view(np.int32)), (name, k)
        res[name] = times
    del multi, singles
    torch.cuda.empty_cache()
    return res


print("card: %s; %d streams" % (card(), S))
d_clip = synth_audio_device(torch, S, 48000, 11, dev)
h_clip = host_array((S, 48000), np.int16, 0)
h_clip[:] = d_clip.cpu().numpy()
d_live = synth_audio_device(torch, S, 480, 12, dev)
for K in (1, 2, 4):
    for name, times in measure(K, d_clip, h_clip, d_live).items():
        m, s = times["multi"], times["separate"]
        print("K=%d %-16s multi %s ms   separate %s ms   (ms per call, rounds; median ratio %.2f)"
              % (K, name, " / ".join("%.2f" % t for t in m), " / ".join("%.2f" % t for t in s), np.median(s) / np.median(m)))
print("card after: %s" % card())
