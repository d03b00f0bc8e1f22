"""tests/detector_cutoffs_ref.py -- TEST INFRASTRUCTURE: both streaming detectors in per-row mode (mww_set_detector_cutoffs,
mww_set_multi_detector_cutoffs of include/mww.h) in NumPy.

RowsRef is the plain detector written out again with a cutoff per row: the same state machine as tests/detector_ref.py,
with float64(avg) > cutoff[r] in place of float64(avg) > cutoff.  ModelsRowsRef is tests/detector_models_ref.py's ModelsRef
with every used model's cutoff held per member row: its update compares float64(avg) elementwise against whatever
self.cutoffs[k] holds, so an array over the rows is the per-row rule for WAKE firing and for the VAD flag alike.

Both start in uniform mode and switch at the first set_cutoffs call with at least one id, every row taking the create-time
cutoff before the listed ones are written; resets keep the cutoffs."""

import numpy as np

from detector_models_ref import OFF, ModelsRef
from detector_ref import EVENT, sort_events


class RowsRef:
    def __init__(self, n_rows, cutoff, window=5, cooldown_slices=25, stream_ids=None):
        self.n_rows, self.window, self.cooldown_slices = int(n_rows), int(window), int(cooldown_slices)
        self.cutoff = float(cutoff)
        self.row_cutoff = None                          # uniform mode
        self.stream_ids = np.arange(n_rows, dtype=np.int32) if stream_ids is None else np.asarray(stream_ids, np.int32)
        self.hist = np.zeros((n_rows, window - 1), np.float32)
        self.seen = np.zeros(n_rows, np.int64)
        self.cooldown = np.full(n_rows, cooldown_slices, np.int32)

    def set_cutoffs(self, rows, cutoffs):
        rows = np.asarray(rows, np.int64).reshape(-1)
        if rows.size == 0:
            return
        if self.row_cutoff is None:
            self.row_cutoff = np.full(self.n_rows, self.cutoff, np.float64)
        self.row_cutoff[rows] = np.broadcast_to(np.asarray(cutoffs, np.float64), rows.shape)

    def cutoffs(self):
        return np.full(self.n_rows, self.cutoff, np.float64) if self.row_cutoff is None else self.row_cutoff.copy()

    def reset(self, rows=None):
        rows = slice(None) if rows is None else [r for r in np.asarray(rows).reshape(-1) if 0 <= r < self.n_rows]
        self.hist[rows] = 0
        self.seen[rows] = 0
        self.cooldown[rows] = self.cooldown_slices

    def update(self, probs):
        """probs [n_rows, n_steps] -> events (EVENT) sorted by (step, stream)"""
        probs = np.asarray(probs, np.float32).reshape(self.n_rows, -1)
        cut = self.cutoffs()
        w, out = self.window, []
        for t in range(probs.shape[1]):
            p = probs[:, t]
            window = np.concatenate([self.hist, p[:, None]], 1)
            s = window[:, 0].copy()
            for j in range(1, w):
                s = (s + window[:, j]).astype(np.float32)       # a sequential float32 sum, oldest first
            avg = (s / np.float32(w)).astype(np.float32)
            full = self.seen + 1 >= w
            cd = np.where(full, np.maximum(self.cooldown - 1, 0), self.cooldown).astype(np.int32)
            fire = full & (cd == 0) & (avg.astype(np.float64) > cut)
            cd[fire] = self.cooldown_slices
            self.cooldown = cd
            rows = np.nonzero(fire)[0]
            ev = np.zeros(rows.size, EVENT)
            ev["stream"], ev["step"], ev["score"] = self.stream_ids[rows], self.seen[rows], avg[rows]
            out.append(ev)
            if w > 1:
                self.hist = window[:, 1:].copy()
            self.seen += 1
        return sort_events(np.concatenate(out) if out else np.zeros(0, EVENT))

    def state(self):
        return dict(hist=self.hist.copy(), seen=self.seen.copy(), cooldown=self.cooldown.copy())


class ModelsRowsRef(ModelsRef):
    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.uniform = list(self.cutoffs)
        self.per_row = False

    def set_cutoffs(self, k, stream_ids, cutoffs):
        """GLOBAL stream ids, members of model k's set"""
        ids = np.asarray(stream_ids, np.int64).reshape(-1)
        if ids.size == 0:
            return
        assert self.roles[k] != OFF and (self.inv[k][ids] >= 0).all()
        if not self.per_row:
            self.cutoffs = [None if r == OFF else np.full(s.size, c, np.float64)
                            for r, s, c in zip(self.roles, self.streams, self.uniform)]
            self.per_row = True
        self.cutoffs[k][self.inv[k][ids]] = np.broadcast_to(np.asarray(cutoffs, np.float64), ids.shape)

    def get_cutoffs(self, k):
        return self.cutoffs[k].copy() if self.per_row else np.full(self.streams[k].size, self.uniform[k], np.float64)
