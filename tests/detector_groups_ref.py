"""NumPy statement of grouped detection (include/mww.h, "grouped detection"), written from the header's rule alone.

GroupRule keeps one window per key (a group, or a (group, model) pair) and takes, at every update, that update's candidates
with (a_u, E_u).  A candidate is a dict with `sample` (its position), `score`, `stream`, `step`, `row` and whatever else the
caller wants carried to the emitted event.  regroup() runs the whole detector: an ungrouped timed detector's events per update,
the rows' groups at that update, and which events are candidates."""

import numpy as np


def better(c, best):
    """the rule's order: highest score, then earliest position, then lowest stream id, then lowest row"""
    if best is None:
        return True
    a = (-float(c["score"]), int(c["sample"]), int(c["stream"]), int(c["row"]))
    b = (-float(best["score"]), int(best["sample"]), int(best["stream"]), int(best["row"]))
    return a < b


class GroupRule:
    def __init__(self, W):
        self.W = int(W)
        self.open = {}                                   # key -> [deadline, best candidate, candidates]

    def _emit(self, key, out):
        D, best, n = self.open.pop(key)
        out.append(dict(best, group=key, candidates=n))

    def update(self, cands, a, E):
        """cands: {key: [candidate, ...]} of this update; a: a_u (None: the update had no step for these keys, step 1 skipped),
        E: E_u (a dict key -> value, or one value for all).  -> the emitted events, each the best candidate with `group` (the
        key) and `candidates`"""
        out = []
        keys = set(self.open) | set(cands)
        for key in sorted(keys, key=repr):
            ak = a[key] if isinstance(a, dict) else a
            Ek = E[key] if isinstance(E, dict) else E
            if key in self.open and ak is not None and ak >= self.open[key][0]:          # step 1
                self._emit(key, out)
            cs = cands.get(key, [])
            if cs:                                                                       # step 2
                if key not in self.open:
                    self.open[key] = [min(int(c["sample"]) for c in cs) + self.W, None, 0]
                w = self.open[key]
                for c in cs:
                    if better(c, w[1]):
                        w[1] = c
                w[2] += len(cs)
            if key in self.open and Ek >= self.open[key][0]:                              # step 3
                self._emit(key, out)
        return out

    def flush(self):
        out = []
        for key in sorted(self.open, key=repr):
            self._emit(key, out)
        return out
