"""tests/detector_ref.py -- TEST INFRASTRUCTURE: the streaming detector in NumPy, one state machine per row held as arrays
over the rows.  Pinned in tests/test_detector.py against tests/golden/detection_golden.npz (the reference's own
compute_false_accepts_per_hour) and oracle/detection_ref.py; the kernels and their host emulation are compared with it.

Per row: hist (the last window - 1 probabilities, oldest first, zeros after a reset), seen, cooldown.  A probability p
arrives: once the row has seen `window` of them, avg = float32 mean of (hist, p) summed oldest first; cooldown =
max(cooldown - 1, 0); the row fires when cooldown == 0 and float64(avg) > cutoff, and then cooldown = cooldown_slices.  The
event's step is `seen` before the increment: the index since reset of the newest probability."""

import numpy as np

EVENT = np.dtype([("stream", np.int32), ("step", np.int64), ("score", np.float32)])


class DetectorRef:
    def __init__(self, n_rows, cutoff, window=5, cooldown_slices=25, stream_ids=None):
        self.n_rows, self.cutoff, self.window, self.cooldown_slices = int(n_rows), float(cutoff), int(window), int(cooldown_slices)
        self.stream_ids = np.arange(n_rows, dtype=np.int32) if stream_ids is None else np.asarray(stream_ids, np.int32)
        self.hist = np.zeros((n_rows, window - 1), np.float32)
        self.seen = np.zeros(n_rows, np.int64)
        self.cooldown = np.full(n_rows, cooldown_slices, np.int32)

    def reset(self, rows=None):
        rows = slice(None) if rows is None else [r for r in np.asarray(rows).reshape(-1) if 0 <= r < self.n_rows]
        self.hist[rows] = 0
        self.seen[rows] = 0
        self.cooldown[rows] = self.cooldown_slices

    def update(self, probs):
        """probs [n_rows, n_steps] -> events (EVENT) sorted by (step, stream)"""
        probs = np.asarray(probs, np.float32).reshape(self.n_rows, -1)
        w, out = self.window, []
        for t in range(probs.shape[1]):
            p = probs[:, t]
            if w > 1:
                s = self.hist[:, 0].copy()
                for j in range(1, w - 1):
                    s = s + self.hist[:, j]                       # float32 + float32: a sequential float32 sum
                s = s + p
            else:
                s = p.copy()
            avg = s / np.float32(w)
            assert avg.dtype == np.float32
            full = self.seen + 1 >= w
            cd = np.where(full, np.maximum(self.cooldown - 1, 0), self.cooldown).astype(np.int32)
            fire = full & (cd == 0) & (avg.astype(np.float64) > self.cutoff)
            cd[fire] = self.cooldown_slices
            self.cooldown = cd
            rows = np.nonzero(fire)[0]
            ev = np.zeros(rows.size, EVENT)
            ev["stream"], ev["step"], ev["score"] = self.stream_ids[rows], self.seen[rows], avg[rows]
            out.append(ev)
            if w > 1:
                self.hist[:, :-1] = self.hist[:, 1:]
                self.hist[:, -1] = p
            self.seen += 1
        ev = np.concatenate(out) if out else np.zeros(0, EVENT)
        return sort_events(ev)

    def state(self):
        return dict(hist=self.hist.copy(), seen=self.seen.copy(), cooldown=self.cooldown.copy())


def sort_events(ev):
    return ev[np.lexsort((ev["stream"], ev["step"]))]


def same_events(a, b):
    """two event arrays (any dtype with stream, step, score) hold the same set, scores as bit patterns"""
    a, b = sort_events(a), sort_events(b)
    return (a.size == b.size and np.array_equal(a["stream"], b["stream"]) and np.array_equal(a["step"], b["step"])
            and np.array_equal(np.ascontiguousarray(a["score"]).view(np.uint32), np.ascontiguousarray(b["score"]).view(np.uint32)))


def same_state(a, b):
    return all(np.array_equal(np.ascontiguousarray(a[k]).view(np.uint8), np.ascontiguousarray(b[k]).view(np.uint8)) for k in ("hist", "seen", "cooldown"))
