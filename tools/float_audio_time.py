"""What float32 device audio costs: a 3 s clip call and a 480-sample live call at 65 536 streams, three ways --
  (a) int16 audio -> predict_clip,
  (b) float32 audio -> predict_clip (converted inside the frontend kernels),
  (c) float32 audio -> torch conversion to int16 (mul, clamp_, copy_ into preallocated buffers) -> int16 predict_clip.
The three arms alternate, each round runs every arm `calls` times, and there are two rounds.  Each arm has its own engine fed the
same audio, so their probabilities must be bit-identical (checked).  Prints the card and its power limit read in the same run.
    python tools/float_audio_time.py [f32|int8] [clip_calls] [live_calls]"""
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import model_blob, synth_audio_device  # noqa: E402
from microwakeword_b200.engine import StreamEngine  # noqa: E402

kind = sys.argv[1] if len(sys.argv) > 1 else "f32"
clip_calls = int(sys.argv[2]) if len(sys.argv) > 2 else 5
live_calls = int(sys.argv[3]) if len(sys.argv) > 3 else 100
S = int(os.environ.get("FLOAT_AUDIO_STREAMS", "65536"))
ROUNDS = 2
dev = torch.device("cuda", 0)


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "%s (nvidia-smi unavailable)" % torch.cuda.get_device_name(0)


def measure(n_samples, calls):
    """-> {arm: [ms per call, one per round]}, {arm: frontend + carry kernel ms per call (library events), last round}"""
    i16 = synth_audio_device(torch, S, n_samples, 11, dev)
    f32 = i16.to(torch.float32).div_(32768.0)           # exact; converts back to the same int16 samples
    tmp_f, tmp_i = torch.empty_like(f32), torch.empty_like(i16)

    def convert_then_int16(eng, out):
        torch.mul(f32, 32768.0, out=tmp_f)
        tmp_f.clamp_(-32768.0, 32767.0)
        tmp_i.copy_(tmp_f)                               # float -> int16 truncates toward zero
        return eng.predict_clip(tmp_i, out=out)

    arms = {"a_int16": lambda eng, out: eng.predict_clip(i16, out=out),
            "b_float32": lambda eng, out: eng.predict_clip(f32, out=out),
            "c_torch_convert": convert_then_int16}
    engines = {k: StreamEngine(model_blob(kind), n_streams=S, device=0) for k in arms}
    outs = {k: torch.empty((S, 128), dtype=torch.float32, device=dev) for k in arms}
    for k, fn in arms.items():                           # warm-up: module load, scratch allocation, steady buffered count
        for _ in range(2):
            fn(engines[k], outs[k])
    torch.cuda.synchronize()
    times, kernels = {k: [] for k in arms}, {}
    last = {}
    for r in range(ROUNDS):
        for k, fn in arms.items():
            eng = engines[k]
            eng.profile(True)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(calls):
                last[k] = fn(eng, outs[k])
            b.record()
            torch.cuda.synchronize()
            p = eng.profile_read()
            eng.profile(False)
            times[k].append(a.elapsed_time(b) / calls)
            kernels[k] = (p["k1_spectral"][0] + p["k2_temporal"][0] + p["carry_update"][0]) / calls
    ref = last["a_int16"].contiguous().view(torch.int32)
    for k in arms:
        assert torch.equal(last[k].contiguous().view(torch.int32), ref), k
    del engines, i16, f32, tmp_f, tmp_i
    torch.cuda.empty_cache()
    return times, kernels


print("card: %s; model %s, %d streams" % (card(), kind, S))
for name, n, calls in (("clip 3 s", 48000, clip_calls), ("live 480", 480, live_calls)):
    times, kernels = measure(n, calls)
    for k in times:
        print("%-9s %-16s call %s ms (rounds)   frontend kernels %.3f ms" % (name, k, " / ".join("%.3f" % t for t in times[k]), kernels[k]))
