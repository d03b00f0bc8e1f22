"""What the media guard costs per poll: the time of one MediaGuard.check (mww_media_check_streams) on a 65 536-stream fp32
okay_nabu engine with a 32 000-sample audio history, n_samples 24 000 (T = 148, 147 words), in two cases:
  * typical ... 32 events, 2 048 ring entries in the window, no registered clip;
  * worst ..... 1 024 events, 16 384 ring entries all in the window, and 16 registered clips of 30 s.
The events are streams of one broadcast (one advert through different gains) and independent streams, half and half, so both
the early-out of non-matching pairs and full lag searches are timed; the ring is filled by earlier checks of the same kind, so
it stays full while timing.  Printed beside a 480-sample live step() of the same engine and a Verifier.verify (fp32
okay_nabu, n_samples 24 000) of the same number of slots.  Times in ms per call from CUDA events, the best of --rounds rounds.
Prints the card, its power limit and the SM clock sampled during the run.  There is no CPU path: without a GPU it fails.
    python tools/media_guard_time.py [--streams 65536] [--rounds 5] [--calls 10]"""
import argparse
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import ClockSampler, model_blob, synth_audio_device  # noqa: E402
from microwakeword_b200.engine import StreamEngine  # noqa: E402
from microwakeword_b200.media import MediaGuard  # noqa: E402
from microwakeword_b200.synth_audio import synth_audio  # noqa: E402
from microwakeword_b200.verify import Verifier  # noqa: E402

HISTORY, N_SAMPLES = 32000, 24000


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "%s (nvidia-smi unavailable)" % torch.cuda.get_device_name(0)


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
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("media_guard_time.py measures the GPU kernels and needs a CUDA device; none is available")
    S, dev = a.streams, torch.device("cuda", 0)
    print("card: %s; %d streams, fp32 okay_nabu, history %d samples, guard n_samples %d" % (card(), S, HISTORY, N_SAMPLES))
    clocks = ClockSampler(0)
    times = {}
    try:
        eng = StreamEngine(model_blob("f32"), n_streams=S)
        eng.set_audio_history(HISTORY)
        P = 1021
        audio = synth_audio_device(torch, P, HISTORY, 3, dev)[torch.arange(S, device=dev) % P].contiguous()
        advert = torch.from_numpy(synth_audio(HISTORY, 77)).to(dev)
        gains = torch.linspace(0.4, 1.2, S // 2, device=dev)[:, None]
        audio[: S // 2] = (advert[None].float() * gains).round().clamp(-32768, 32767).to(torch.int16)
        probs = torch.empty((S, 1), dtype=torch.float32, device=dev)
        for i in range(HISTORY // 480):
            eng.step(audio[:, 480 * i:480 * (i + 1)].contiguous(), out=probs)
        chunk = audio[:, :480].contiguous()
        step = lambda: eng.step(chunk, out=probs)                                  # noqa: E731
        step()
        times["step() 480 samples"] = [event_time(step, 50) for _ in range(a.rounds)]
        end = eng.audio_samples_seen
        gen = np.random.default_rng(0)
        for name, n, ring, clips in (("typical", 32, 2048, 0), ("worst", 1024, 16384, 16)):
            guard = MediaGuard(slots=n, ring=ring, max_media=max(clips, 1), max_media_s=30)
            for k in range(clips):
                guard.register(synth_audio(30 * 16000, 500 + k))
            half = n // 2
            # independent slots on distinct base streams: stream s carries base s % P, and S / 2 + k for distinct k < P differ mod P
            ind = S // 2 + gen.choice(P, n - half, replace=False)
            ids = np.concatenate([gen.choice(S // 2, half, replace=False), ind]).astype(np.int32)
            ids_d = torch.from_numpy(ids).to(dev)
            ends = torch.full((n,), end, dtype=torch.int64, device=dev)
            fn = (lambda guard=guard, ids_d=ids_d, ends=ends: guard.check(eng, ids_d, ends=ends))
            for _ in range(ring // n + 1):                                         # fill the ring
                fn()
            info = guard.info()
            times["check %s: %d events, %d ring entries, %d clips" % (name, n, info.ring_fill, info.n_media)] = \
                [event_time(fn, a.calls) for _ in range(a.rounds)]
            ver = Verifier(model_blob("f32"), slots=n, n_samples=N_SAMPLES, cutoff=0.5)
            vfn = (lambda ver=ver, ids_d=ids_d: ver.verify(eng, ids_d))
            vfn()
            times["verify %d slots" % n] = [event_time(vfn, a.calls) for _ in range(a.rounds)]
            m = guard.check(eng, ids_d, ends=ends)[1].cpu().numpy()
            print("%s: flagged %d of %d broadcast slots and %d of %d independent ones" % (name, (m[:half] != 0).sum(), half, (m[half:] != 0).sum(), n - half))
            guard.close()
            ver.close()
            torch.cuda.empty_cache()
    finally:
        sampled = clocks.stop()
    print("SM clock during the run: median %s MHz (max %s MHz), throttle reasons seen: %s" %
          (sampled["sm_mhz"], sampled["sm_max_mhz"], ", ".join(sampled["reasons"]) or "none"))
    for k, t in times.items():
        print("%-58s best %8.3f ms per call (rounds %s)" % (k, min(t), " / ".join("%.3f" % x for x in t)))


if __name__ == "__main__":
    main()
