"""What grouped detection costs: a grouped against an ungrouped timed StreamDetector update at --rows rows in --groups households of
one to four rows, 1 and 100 steps per call (the thread and the warp form).  Two probability sets: every row's cutoff above any
average (no event: the cost of the grouped path and of the close over every group), and household-correlated probabilities
a cutoff of 0.75 (the offers' atomics included; drained between rounds, outside the timing; the events of one call printed).
Times in ms per call from CUDA events, the best of --rounds rounds, each pair alternated in the same round.  Prints the card,
its power limit and the SM clock sampled during the run.  There is no CPU path: without a GPU it fails.
    python tools/detector_groups_time.py [--rows 65536] [--groups 16384] [--rounds 5]"""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench import ClockSampler  # noqa: E402
from event_positions_time import card, event_time  # noqa: E402
from microwakeword_b200.detection import StreamDetector  # noqa: E402


class Clock:
    """one engine call's counters, held still: every update is described by the same clock (the windows of a grouped
    detector then close at the next update, W being below one step)"""

    def __init__(self, S):
        self.S, self.hop, self.frontend_buffered, self.stride, self.pending_rows = S, 160, 320, 3, 0

    def _audio_history(self):
        return 1, self.S


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--rows", type=int, default=65536)
    ap.add_argument("--groups", type=int, default=16384)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("detector_groups_time.py needs a CUDA device (there is no CPU path)")
    print("card: %s" % card())
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(1)
    sizes = rng.integers(1, 5, a.groups)
    groups = np.full(a.rows, -1, np.int32)
    members = np.repeat(np.arange(a.groups), sizes)[:a.rows]
    groups[rng.permutation(a.rows)[:members.size]] = members
    gidx = torch.from_numpy(np.where(groups < 0, a.groups, groups).astype(np.int64)).to(dev)
    clock = Clock(48000 * 60)
    clocks = ClockSampler(0)
    try:
        for label, cut in (("no event", 2.0), ("events", 0.75)):
            plain = StreamDetector(a.rows, cut, capacity=1 << 20, timed=True)
            grouped = StreamDetector(a.rows, cut, capacity=1 << 20, timed=True, groups=a.groups, group_window=240)
            grouped.set_groups(np.arange(a.rows), groups)
            for steps in (1, 100):
                hh = torch.rand(a.groups + 1, steps, device=dev)
                p = (0.6 * hh[gidx] + 0.4 * torch.rand(a.rows, steps, device=dev)).contiguous()
                up, ug = (lambda: plain.update(p, clock)), (lambda: grouped.update(p, clock))
                up(), ug()
                torch.cuda.synchronize()
                tp, tg = [], []
                for _ in range(a.rounds):
                    tp.append(event_time(up, a.calls))
                    tg.append(event_time(ug, a.calls))
                    plain.drain(), grouped.drain()
                up(), ug()
                torch.cuda.synchronize()
                ev, eg = int(plain.event_count.item()), int(grouped.event_count.item())
                plain.drain(), grouped.drain()
                print("%s: %d rows, %d groups, %3d steps: ungrouped timed %.4f ms, grouped %.4f ms  (events of one call: %d ungrouped, %d grouped)"
                      % (label, a.rows, a.groups, steps, min(tp), min(tg), ev, eg))
            plain.close()
            grouped.close()
    finally:
        print("SM clock during the run: %s" % clocks.stop())


if __name__ == "__main__":
    main()
