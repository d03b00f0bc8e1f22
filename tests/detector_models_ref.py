"""tests/detector_models_ref.py -- TEST INFRASTRUCTURE: the multi-model streaming detector (mww_multi_detector_create,
include/mww.h) in NumPy.  Every model's rows are arrays over the members of its stream set, in list order; an update
takes each model's probabilities of one handle call with the call's step counts n_k and the pending rows p_k before it.

Step j of model k ends at call-relative feature row e_k(j) = (j + 1) s_k - p_k - 1.  Every stream walks its steps in order
of e, a VAD step before a WAKE step that ends on the same row; since e does not depend on the stream, one global order
serves all of them and each step runs over all rows of its model at once.  A VAD step sets active = (seen >= window and
float64(avg) > cutoff), seen counting this step.  A WAKE step is tests/detector_ref.py's rule, firing only where the
stream's VAD row is active (always when there is no VAD, never for a stream the VAD does not score)."""

import numpy as np

OFF, WAKE, VAD = 0, 1, 2
MEVENT = np.dtype([("stream", np.int32), ("model", np.int32), ("step", np.int64), ("score", np.float32)])


def call_steps(strides, pending, rows):
    """what a handle call of `rows` new feature rows does to models of the given strides holding `pending` rows:
    (steps per model, pending rows after)"""
    return [(p + rows) // s for p, s in zip(pending, strides)], [(p + rows) % s for p, s in zip(pending, strides)]


def call_fits(roles, strides, n_steps, pending):
    """whether one R >= 0 gives every non-OFF model n_k = (p_k + R) div s_k with 0 <= p_k < s_k (searched, not solved)"""
    used = [k for k in range(len(roles)) if roles[k] != OFF]
    if any(n_steps[k] < 0 or not 0 <= pending[k] < strides[k] for k in used):
        return False
    top = max((n_steps[k] + 1) * strides[k] for k in used)
    return any(all((pending[k] + R) // strides[k] == n_steps[k] for k in used) for R in range(top + 1))


def sort_model_events(ev):
    return ev[np.lexsort((ev["stream"], ev["step"], ev["model"]))]


def same_model_events(a, b):
    """two event arrays (any dtype with stream, model, step, score) hold the same set, scores as bit patterns"""
    a, b = sort_model_events(a), sort_model_events(b)
    return (a.size == b.size and all(np.array_equal(a[f], b[f]) for f in ("stream", "model", "step"))
            and np.array_equal(np.ascontiguousarray(a["score"]).view(np.uint32), np.ascontiguousarray(b["score"]).view(np.uint32)))


def same_model_state(a, b):
    """two state lists (None for an OFF model, else dict of arrays) bit for bit"""
    if len(a) != len(b):
        return False
    for x, y in zip(a, b):
        if (x is None) != (y is None):
            return False
        if x is not None and (x.keys() != y.keys() or not all(
                np.array_equal(np.ascontiguousarray(x[f]).view(np.uint8), np.ascontiguousarray(y[f]).view(np.uint8)) for f in x)):
            return False
    return True


class ModelsRef:
    def __init__(self, n_streams, roles, windows, cutoffs, cooldowns, strides, streams=None):
        K = len(roles)
        self.n_streams, self.K = int(n_streams), K
        self.roles, self.windows, self.strides = list(roles), [int(w) for w in windows], [int(s) for s in strides]
        self.cutoffs, self.cooldowns = [float(c) for c in cutoffs], [int(c) for c in cooldowns]
        self.streams = [np.arange(n_streams, dtype=np.int32) if streams is None or streams[k] is None else np.asarray(streams[k], np.int32)
                        for k in range(K)]
        self.vad = next((k for k in range(K) if roles[k] == VAD), None)
        self.inv = []
        for k in range(K):
            inv = np.full(n_streams, -1, np.int64)
            inv[self.streams[k]] = np.arange(self.streams[k].size)
            self.inv.append(inv)
        self.hist = [np.zeros((s.size, w - 1), np.float32) for s, w in zip(self.streams, self.windows)]
        self.seen = [np.zeros(s.size, np.int64) for s in self.streams]
        self.flag = [np.zeros(s.size, np.int32) for s in self.streams]
        self.reset()

    def reset(self, ids=None):
        """fresh state of every used model for all streams (None) or the given global ids (out of range ignored)"""
        for k in range(self.K):
            if self.roles[k] == OFF:
                continue
            if ids is None:
                rows = slice(None)
            else:
                g = np.asarray(ids, np.int64).reshape(-1)
                g = g[(g >= 0) & (g < self.n_streams)]
                rows = self.inv[k][g]
                rows = rows[rows >= 0]
            self.hist[k][rows] = 0
            self.seen[k][rows] = 0
            self.flag[k][rows] = self.cooldowns[k] if self.roles[k] == WAKE else 0

    def _push(self, k, p):
        """float32 mean of (history, p), summed oldest first; p joins the history"""
        h, w = self.hist[k], self.windows[k]
        if w > 1:
            s = h[:, 0].copy()
            for j in range(1, w - 1):
                s = s + h[:, j]
            s = s + p
            h[:, :-1] = h[:, 1:]
            h[:, -1] = p
        else:
            s = p.copy()
        avg = s / np.float32(w)
        assert avg.dtype == np.float32
        return avg

    def _gate(self, k):
        """the VAD flag of each row of WAKE model k's streams"""
        if self.vad is None:
            return np.ones(self.streams[k].size, bool)
        vr = self.inv[self.vad][self.streams[k]]
        return np.where(vr >= 0, self.flag[self.vad][np.maximum(vr, 0)] != 0, False)

    def update(self, probs, n_steps, pending):
        """probs[k]: [members of model k, >= n_steps[k]] (None for OFF); -> events (MEVENT) sorted by (model, step, stream)"""
        assert call_fits(self.roles, self.strides, n_steps, pending), (n_steps, pending)
        order = []
        for k in range(self.K):
            if self.roles[k] == OFF:
                continue
            for j in range(n_steps[k]):
                order.append(((j + 1) * self.strides[k] - pending[k] - 1, 0 if self.roles[k] == VAD else 1, k, j))
        out = []
        for _, _, k, j in sorted(order):
            p = np.asarray(probs[k], np.float32)[:, j]
            avg = self._push(k, p)
            self.seen[k] += 1
            full = self.seen[k] >= self.windows[k]
            if self.roles[k] == VAD:
                self.flag[k] = (full & (avg.astype(np.float64) > self.cutoffs[k])).astype(np.int32)
                continue
            cd = np.where(full, np.maximum(self.flag[k] - 1, 0), self.flag[k]).astype(np.int32)
            fire = full & (cd == 0) & (avg.astype(np.float64) > self.cutoffs[k]) & self._gate(k)
            cd[fire] = self.cooldowns[k]
            self.flag[k] = cd
            rows = np.nonzero(fire)[0]
            ev = np.zeros(rows.size, MEVENT)
            ev["stream"], ev["model"], ev["step"], ev["score"] = self.streams[k][rows], k, self.seen[k][rows] - 1, avg[rows]
            out.append(ev)
        return sort_model_events(np.concatenate(out) if out else np.zeros(0, MEVENT))

    def state(self):
        """per model: None (OFF) or {hist, seen, cooldown | active}, rows in list order"""
        return [None if r == OFF else {"hist": h.copy(), "seen": s.copy(), ("active" if r == VAD else "cooldown"): f.copy()}
                for r, h, s, f in zip(self.roles, self.hist, self.seen, self.flag)]


def feed(det, seqs, strides, pending0, row_calls, resets=None):
    """Run `det` (ModelsRef or anything with its update) over whole per-model probability sequences seqs[k] ([members,
    >= total steps]; None for OFF) as handle calls of row_calls[c] feature rows each, starting from pending0.  resets:
    {call index: ids} -- det.reset(ids) before that call.  -> concatenated events, pending rows after the last call."""
    pending, at, evs = list(pending0), [0] * len(strides), []
    for c, rows in enumerate(row_calls):
        if resets and c in resets:
            det.reset(resets[c])
        n, after = call_steps(strides, pending, rows)
        probs = [None if s is None else s[:, a:a + m] for s, a, m in zip(seqs, at, n)]
        evs.append(det.update(probs, n, pending))
        at = [a + m for a, m in zip(at, n)]
        pending = after
    return (np.concatenate(evs) if evs else np.zeros(0, MEVENT)), pending
