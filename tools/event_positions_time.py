"""What event positions cost: a timed against an untimed detector update, and the anchored against the "now" verify.
  * update: StreamDetector.update at --rows rows of random probabilities, 1 and 100 steps per call (the thread and the warp
    form), untimed (mww_detector_update) and timed (mww_update_detector_at); and the same for a MultiModelDetector over a
    two-model engine of --rows streams (mww_multi_detector_update against mww_update_multi_detector_at), the probabilities
    of one engine call of 480 and of 48 000 samples.  Every row's cutoff is 2, so no event fires: the time is the rule's.
  * verify at --slots slots of a 65 536-stream fp32 okay_nabu engine: the "now" verify with n_samples = 32 000 + 33 x 480
    (what a server that drains once a second must read) against the anchored verify with n_samples = 32 000 and post = 3 200.
Times in ms per call from CUDA events, the best of --rounds rounds, each pair alternated in the same round.  Prints the card,
its power limit and the SM clock sampled during the run.  There is no CPU path: without a GPU it fails.
    python tools/event_positions_time.py [--rows 65536] [--slots 1024] [--rounds 5]"""
import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import ClockSampler, model_blob, synth_audio_device  # noqa: E402
from microwakeword_b200.detection import MultiModelDetector, StreamDetector  # noqa: E402
from microwakeword_b200.engine import MultiModelEngine, StreamEngine  # noqa: E402
from microwakeword_b200.verify import Verifier  # noqa: E402


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


def best_pair(a, b, rounds, calls):
    """(best ms of a, best ms of b), alternated round by round"""
    a(), b()
    torch.cuda.synchronize()
    ta, tb = [], []
    for _ in range(rounds):
        ta.append(event_time(a, calls))
        tb.append(event_time(b, calls))
    return min(ta), min(tb)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--rows", type=int, default=65536)
    ap.add_argument("--slots", type=int, default=1024)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("event_positions_time.py needs a CUDA device (there is no CPU path)")
    print("card: %s" % card())
    dev = torch.device("cuda", 0)
    blob = model_blob("f32")
    clocks = ClockSampler(0)
    try:
        eng = StreamEngine(blob, n_streams=a.rows)
        eng.set_audio_history(48000)
        eng.step(synth_audio_device(torch, a.rows, 480, 1, dev))
        plain, timed = StreamDetector(a.rows, 2.0, capacity=1024), StreamDetector(a.rows, 2.0, capacity=1024, timed=True)
        for steps in (1, 100):
            p = torch.rand(a.rows, steps, device=dev)
            u, t = best_pair(lambda: plain.update(p), lambda: timed.update(p, eng), a.rounds, a.calls)
            print("plain update, %d rows, %3d steps: untimed %.4f ms, timed %.4f ms" % (a.rows, steps, u, t))
        del eng
        meng = MultiModelEngine([blob, blob], n_streams=a.rows)
        meng.set_audio_history(48000)
        meng.predict_clip(synth_audio_device(torch, a.rows, 960, 2, dev))
        for n in (480, 48000):
            probs = meng.predict_clip(synth_audio_device(torch, a.rows, n, 2, dev))
            probs = [torch.rand_like(q) for q in probs]
            mp = MultiModelDetector(meng, cutoffs=[2.0, 2.0], capacity=1024)
            mt = MultiModelDetector(meng, cutoffs=[2.0, 2.0], capacity=1024, timed=True)
            # the same call described again: the engine's counters stand still, so both detectors accept it every time
            pend = list(meng.pending_rows)

            def untimed():
                mp._pending = list(pend)
                mp.update(probs)

            def timed_models():
                mt._pending = list(pend)
                mt.update(probs)
            u, t = best_pair(untimed, timed_models, a.rounds, a.calls)
            print("models update, %d streams x 2 models, %3d steps: untimed %.4f ms, timed %.4f ms" % (a.rows, probs[0].shape[1], u, t))
        del meng
        src = StreamEngine(blob, n_streams=65536)
        src.set_audio_history(48000)
        x = synth_audio_device(torch, 65536, 480 * 120, 3, dev)
        det = StreamDetector(65536, -1.0, capacity=a.slots, timed=True)          # every slot used
        for i in range(120):
            det.update(src.step(x[:, 480 * i:480 * (i + 1)].contiguous()), src)
        now = Verifier(blob, slots=a.slots, n_samples=32000 + 33 * 480, cutoff=0.5)
        at = Verifier(blob, slots=a.slots, n_samples=32000, cutoff=0.5)
        u, t = best_pair(lambda: now.verify(src, det), lambda: at.verify(src, det, at_event=True, post=3200), a.rounds, 5)
        print("verify, %d slots: now (n_samples %d) %.3f ms, at the event (n_samples 32000, post 3200) %.3f ms"
              % (a.slots, 32000 + 33 * 480, u, t))
    finally:
        print("SM clock during the run: %s" % clocks.stop())


if __name__ == "__main__":
    main()
