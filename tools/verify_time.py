"""What one second-stage verification costs: the time of one Verifier.verify call (mww_verify_streams over `slots` stream ids
of a 65 536-stream fp32 okay_nabu engine with a 32 000-sample audio history) at --slots 64 / 256 / 1024 and n_samples 32 000
(2 s), with two verifier models:
  * okay_nabu ... the fp32 okay_nabu container (tests/golden/okay_nabu_synth_f32.mww), on the tensor-core clip kernels;
  * wide ........ an fp32 model of a wider run-time geometry (the `wide` geometry of tests/generic_range.py: 512 first-conv
                  filters, blocks of 257, 129 and 512 channels), on the run-time-geometry kernels.
Printed beside what the live loop of the same engine costs per 30 ms: one 480-sample step() call and one
StreamDetector.update() of its probabilities.  A verify call runs the verifier on all of its slots whatever the number of
events, so its time does not depend on how many streams fired.  Times in ms per call from CUDA events, the best of --rounds
rounds.  Prints the card, its power limit and the SM clock sampled during the run.  There is no CPU path: without a GPU it
fails.
    python tools/verify_time.py [--streams 65536] [--slots 64 256 1024] [--rounds 5]"""
import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import ClockSampler, model_blob, synth_audio_device  # noqa: E402
from microwakeword_b200 import model_file as MF  # noqa: E402
from microwakeword_b200.detection import StreamDetector  # noqa: E402
from microwakeword_b200.engine import StreamEngine  # noqa: E402
from microwakeword_b200.verify import Verifier  # noqa: E402

P = 1021                         # distinct base streams; stream s carries base[s % P]
N_SAMPLES = 32000


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "%s (nvidia-smi unavailable)" % torch.cuda.get_device_name(0)


def wide_blob():
    from oracle import mixednet_ref as R          # synthetic weights of the test geometry (NumPy only)
    spec = R.Spec(512, 5, 3, (257, 129, 512), ((3, 5, 7, 9), (1, 11), (5,)), head_rows=8)
    return MF.write_container(R.fold_bn(spec, R.init_synthetic(spec, 0)))


def event_time(fn, calls):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(calls):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / calls


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--streams", type=int, default=65536)
    ap.add_argument("--slots", type=int, nargs="+", default=[64, 256, 1024])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("verify_time.py measures the GPU kernels and needs a CUDA device; none is available")
    S = a.streams
    print("card: %s; %d streams, fp32 okay_nabu, history %d samples, verifier n_samples %d" % (card(), S, N_SAMPLES, N_SAMPLES))
    clocks = ClockSampler(0)
    try:
        eng = StreamEngine(model_blob("f32"), n_streams=S)
        eng.set_audio_history(N_SAMPLES)
        idx = torch.arange(S, device="cuda") % P
        audio = synth_audio_device(torch, P, N_SAMPLES + 480, 3, torch.device("cuda", 0))[idx].contiguous()
        probs = torch.empty((S, 1), dtype=torch.float32, device="cuda")
        for i in range(N_SAMPLES // 480):            # fill the history
            eng.step(audio[:, 480 * i:480 * (i + 1)], out=probs)
        chunk = audio[:, :480].contiguous()
        det = StreamDetector(S, cutoff=2.0, capacity=max(a.slots))       # a cutoff no average reaches: the update's own cost
        live = {"step() 480 samples": lambda: eng.step(chunk, out=probs), "StreamDetector.update()": lambda: det.update(probs)}
        times = {k: [] for k in live}
        for k, fn in live.items():
            fn()
        for _ in range(a.rounds):
            for k, fn in live.items():
                times[k].append(event_time(fn, 50))
        blobs = {"okay_nabu": model_blob("f32"), "wide": wide_blob()}
        gen = torch.Generator(device="cuda").manual_seed(0)
        for slots in a.slots:
            ids = torch.randperm(S, device="cuda", generator=gen)[:slots].to(torch.int32)
            for name, blob in blobs.items():
                ver = Verifier(blob, slots=slots, n_samples=N_SAMPLES, cutoff=0.5)
                fn = (lambda ver=ver, ids=ids: ver.verify(eng, ids))
                fn()
                key = "verify %s, %d slots" % (name, slots)
                times[key] = [event_time(fn, a.calls) for _ in range(a.rounds)]
                ver.close()
                torch.cuda.empty_cache()
    finally:
        sampled = clocks.stop()
    print("SM clock during the run: median %s MHz (max %s MHz), throttle reasons seen: %s" %
          (sampled["sm_mhz"], sampled["sm_max_mhz"], ", ".join(sampled["reasons"]) or "none"))
    for k, t in times.items():
        print("%-32s best %8.3f ms per call (rounds %s)" % (k, min(t), " / ".join("%.3f" % x for x in t)))


if __name__ == "__main__":
    main()
