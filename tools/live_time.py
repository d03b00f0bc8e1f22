"""Timing of the live-step path only (65 536 streams, 480 samples per call): per-kernel ms from the library's CUDA events.
    python tools/live_time.py [f32|int8] [calls]"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import measured_peaks, model_blob, synth_audio_device  # noqa: E402
from microwakeword_b200.engine import StreamEngine  # noqa: E402

kind = sys.argv[1] if len(sys.argv) > 1 else "f32"
calls = int(sys.argv[2]) if len(sys.argv) > 2 else 60
S = int(os.environ.get("LIVE_STREAMS", "65536"))
dev = torch.device("cuda", 0)
eng = StreamEngine(model_blob(kind), n_streams=S, device=0)
audio = synth_audio_device(torch, S, 480 * 8, 5, dev)
chunks = [audio[:, 480 * i:480 * (i + 1)].contiguous() for i in range(8)]
probs = torch.empty((S, 2), dtype=torch.float32, device=dev)
for c in chunks[:4]:
    eng.predict_clip(c, out=probs)
torch.cuda.synchronize()
eng.profile(True)
a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
a.record()
for i in range(calls):
    eng.predict_clip(chunks[i % 8], out=probs)
b.record()
torch.cuda.synchronize()
p = eng.profile_read()
eb = 4 if kind == "f32" else 1
step_bytes = 4176 * eb + 368 * eb + 240 + 4
nn = p["mixednet"][0] / max(p["mixednet"][1], 1)
peak, peak_src = measured_peaks()
print("%s mode=%s variant=%s: call %.4f ms, frontend %.4f, nn %.4f ms = %.0f GB/s (%.3f of %.0f GB/s, %s)" % (
    kind, os.environ.get("MWW_LIVE_MODE", "0"), os.environ.get("MWW_LIVE_VARIANT", "-"), a.elapsed_time(b) / calls, p["k1_spectral"][0] / calls, nn,
    S * step_bytes / nn / 1e6, S * step_bytes / nn / 1e6 / peak, peak, peak_src))
