"""The playback guard's rule (include/mww.h, "playback guard") stated in NumPy, independently of the C bodies: each stream's
playback pb_s as a plain array over a window of the history axis, rows as a set of held streams with heads, the release at
every write call, MWW_ENOMEM, reads, the heard rule and the decision."""

import numpy as np

ENOMEM = -4


class Rule:
    def __init__(self, n_streams, rows, C, lo=-(1 << 18), hi=1 << 20):
        self.n_streams, self.rows, self.C, self.lo, self.size = n_streams, rows, C, lo, hi - lo
        self.pb = {}                                         # stream -> pb_s(p) at index p - lo, for the streams ever written
        self.head = {}                                       # stream -> w, for the streams that hold a row

    def write(self, ids, starts, x, seen):
        """one write call at samples_seen = seen; returns 0, or ENOMEM with nothing changed"""
        C = self.C
        kept = {s: w for s, w in self.head.items() if w > seen - C}          # the release
        if len(kept) + sum(1 for s in ids if s not in kept) > self.rows:
            return ENOMEM
        self.head = kept
        for s, a, row in zip(ids, starts, x):
            s, a = int(s), int(a)
            if s not in self.head:                                         # a fresh row: zeros, head a - C
                self.pb[s] = np.zeros(self.size, np.int16)
                self.head[s] = a - C
            w = self.head[s]
            n = len(row)
            w2 = max(w, a + n)
            if a > w:
                self.pb[s][w - self.lo:a - self.lo] = 0
            self.pb[s][a - self.lo:a + n - self.lo] = row
            self.head[s] = w2
        return 0

    def reset(self, ids=None):
        if ids is None:
            self.head = {}
        for s in ids if ids is not None else ():
            self.head.pop(int(s), None)

    def read(self, s, end, n):
        """pb_s over [end - n, end) as the row holds it"""
        out = np.zeros(n, np.int16)
        if s not in self.head:
            return out
        w = self.head[s]
        p = np.arange(end - n, end)
        held = (p >= w - self.C) & (p < w)
        out[held] = self.pb[s][p[held] - self.lo]
        return out

    def heard(self, s, r0, seen):
        if not 0 <= s < self.n_streams or s not in self.head:
            return False
        w = self.head[s]
        return r0 >= seen - self.C and r0 >= w - self.C and r0 < w


def decide(heard, score, cutoff, confirmed):
    """(score, flagged, passed) of one slot"""
    if not heard:
        return np.float32(np.nan), 0, confirmed
    flagged = float(score) > cutoff
    return np.float32(score), int(flagged), -1 if flagged else confirmed
