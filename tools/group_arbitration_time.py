"""What group arbitration costs: an arbitrated against a score-grouped timed StreamDetector update at --rows rows in --groups
households of one to four rows, with live (1-step) and 100-step calls, on a StreamEngine whose audio history the arbitrated
detector measures (Ls + Ln = 12 000 + 8 000 samples read per candidate).  Three cases: no event; about 32 candidates per update
(32 grouped rows fire at one step of the call); a wave (every grouped row fires at one step of the call).  Window 1, cooldown 0
and a window below one step, so every call offers and closes the same way.  Times in ms per call from CUDA events, the best of
--rounds rounds, the pair alternated in each round; drained between rounds, outside the timing.  Prints the card, its power
limit and the SM clock sampled during the run.  There is no CPU path: without a GPU it fails.
    python tools/group_arbitration_time.py [--rows 65536] [--groups 16384] [--rounds 5]"""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench import ClockSampler, model_blob, synth_audio_device  # noqa: E402
from event_positions_time import card, event_time  # noqa: E402
from microwakeword_b200.detection import StreamDetector  # noqa: E402
from microwakeword_b200.engine import StreamEngine  # noqa: E402


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--rows", type=int, default=65536)
    ap.add_argument("--groups", type=int, default=16384)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("group_arbitration_time.py needs a CUDA device (there is no CPU path)")
    print("card: %s" % card())
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(1)
    sizes = rng.integers(1, 5, a.groups)
    groups = np.full(a.rows, -1, np.int32)
    members = np.repeat(np.arange(a.groups), sizes)[:a.rows]
    groups[rng.permutation(a.rows)[:members.size]] = members
    grouped_rows = np.flatnonzero(groups >= 0)
    eng = StreamEngine(model_blob("f32"), n_streams=a.rows)
    eng.set_audio_history(48000)
    base = synth_audio_device(torch, 1021, 480 * 100, 3, dev)[torch.arange(a.rows, device=dev) % 1021]
    for i in range(100):                                   # 3 s of audio in every ring
        eng.step(base[:, 480 * i:480 * (i + 1)].contiguous())
    del base
    clocks = ClockSampler(0)
    try:
        score = StreamDetector(a.rows, 0.5, window=1, cooldown_slices=0, capacity=1 << 20, timed=True, groups=a.groups, group_window=240)
        arb = StreamDetector(a.rows, 0.5, window=1, cooldown_slices=0, capacity=1 << 20, timed=True, groups=a.groups, group_window=240)
        for d in (score, arb):
            d.set_groups(np.arange(a.rows), groups)
        arb.arbitrate(eng, 12000, 8000)
        firing = {"no event": np.zeros(0, np.int64), "32 candidates": rng.choice(grouped_rows, 32, replace=False), "wave": grouped_rows}
        for label, rows in firing.items():
            for steps in (1, 100):
                p = torch.zeros(a.rows, steps, device=dev)
                p[torch.from_numpy(rows).to(dev), steps - 1] = 1.0
                us, ua = (lambda: score.update(p, eng)), (lambda: arb.update(p, eng))
                us(), ua()
                torch.cuda.synchronize()
                score.drain(), arb.drain()
                ts, ta = [], []
                for _ in range(a.rounds):
                    ts.append(event_time(us, a.calls))
                    ta.append(event_time(ua, a.calls))
                    score.drain(), arb.drain()
                us(), ua()
                torch.cuda.synchronize()
                es, ea = int(score.event_count.item()), int(arb.event_count.item())
                score.drain(), arb.drain()
                print("%s: %d rows, %d groups, %3d steps: score-grouped %.4f ms, arbitrated %.4f ms  (candidates of one call: %d; events: %d, %d)"
                      % (label, a.rows, a.groups, steps, min(ts), min(ta), rows.size, es, ea))
        score.close()
        arb.close()
    finally:
        print("SM clock during the run: %s" % clocks.stop())
        eng.close()


if __name__ == "__main__":
    main()
