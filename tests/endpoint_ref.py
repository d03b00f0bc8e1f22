"""tests/endpoint_ref.py -- TEST INFRASTRUCTURE: the endpointer (mww_endpointer_*, include/mww.h "endpointing") in NumPy,
written from the rule text.  Rows are the members of the model's stream set in list order; an update takes the model's
probabilities of one handle call with the handle's counters read right after it (samples_seen S, frontend_buffered and the
model's pending rows g), and places step j at pos(j) = S - b - hop (g + (n - 1 - j) s), b = buffered - (480 - hop)."""

import numpy as np

END_OF_SPEECH, NO_SPEECH, MAX_LENGTH = 1, 2, 3
EVENT = np.dtype([("stream", np.int32), ("reason", np.int32), ("start_sample", np.int64), ("end_sample", np.int64),
                  ("speech_end_sample", np.int64), ("steps", np.int32), ("pad", np.int32)])
ROW_FIELDS = ("seen", "flags", "armed", "elapsed", "run", "silence", "heard", "start_sample", "speech_end_sample")
SEG = ("elapsed", "run", "silence", "heard", "start_sample", "speech_end_sample")


def position(S, buffered, hop, pending, stride, n, j):
    b = buffered - (480 - hop)
    return S - b - hop * (pending + (n - 1 - j) * stride)


def update_fits(S0, buffered0, pending0, S, buffered, pending, hop, stride, n):
    moved = (S - buffered) - (S0 - buffered0)
    if moved < 0 or moved % hop or n < 0 or not 0 <= pending < stride:
        return False
    return n * stride == pending0 + moved // hop - pending


class EndpointRef:
    def __init__(self, n_streams, members, stride, hop, vad_window=5, vad_cutoff=0.5, speech_steps=3, silence_steps=25, timeout_steps=100,
                 max_steps=334, lookback_steps=64, capacity=64, counters=(0, 0, 0)):
        self.n_streams, self.members = n_streams, np.asarray(members, np.int32)
        self.stride, self.hop, self.w, self.cutoff = stride, hop, vad_window, float(vad_cutoff)
        self.speech_steps, self.silence_steps, self.timeout_steps, self.max_steps = speech_steps, silence_steps, timeout_steps, max_steps
        self.lookback, self.capacity = lookback_steps, capacity
        self.row_of = np.full(n_streams, -1, np.int64)
        self.row_of[self.members] = np.arange(self.members.size)
        R = self.members.size
        self.hist = np.zeros((R, vad_window - 1), np.float32)
        self.rows = {k: np.zeros(R, np.uint64 if k == "flags" else np.int64) for k in ROW_FIELDS}
        self.rows["armed"][:] = -1
        self.base = tuple(counters)
        self.steps, self.positions = 0, []            # positions of every step consumed, oldest first
        self.events, self.count = [], 0

    # ---- segmenter, over an index array of rows at once ----
    def _fresh(self, rows):
        for k in SEG:
            self.rows[k][rows] = 0

    def _segment(self, rows, f, p):
        """one step of the listed rows with flags f at position p -> reason per row (0: goes on)"""
        g = self.rows
        first = rows[g["elapsed"][rows] == 0]
        g["start_sample"][first] = g["speech_end_sample"][first] = p - self.stride * self.hop
        g["elapsed"][rows] += 1
        on, off = rows[f], rows[~f]
        g["run"][on] += 1
        g["silence"][on] = 0
        g["heard"][on[g["run"][on] >= self.speech_steps]] = 1
        g["speech_end_sample"][on[g["heard"][on] == 1]] = p
        g["run"][off] = 0
        g["silence"][off] += 1
        heard = g["heard"][rows] == 1
        reason = np.where(heard & (g["silence"][rows] >= self.silence_steps), END_OF_SPEECH,
                          np.where(~heard & (g["elapsed"][rows] >= self.timeout_steps), NO_SPEECH,
                                   np.where(g["elapsed"][rows] >= self.max_steps, MAX_LENGTH, 0)))
        return reason

    def _end(self, rows, reasons, p):
        g = self.rows
        for r, reason in zip(rows, reasons):
            e = (int(self.members[r]), int(reason), int(g["start_sample"][r]), int(p), int(g["speech_end_sample"][r]), int(g["elapsed"][r]), 0)
            if self.count < self.capacity:
                self.events.append(e)
            self.count += 1
        g["armed"][rows] = -1
        self._fresh(rows)

    # ---- calls ----
    def update(self, probs, S, buffered, pending):
        probs = np.asarray(probs, np.float32)
        n = probs.shape[1]
        if not update_fits(*self.base, S, buffered, pending, self.hop, self.stride, n):
            raise ValueError("inconsistent update")
        self.base = (S, buffered, pending)
        g = self.rows
        for j in range(n):
            p = position(S, buffered, self.hop, pending, self.stride, n, j)
            col = probs[:, j]
            s = self.hist[:, 0].copy() if self.w > 1 else col.copy()
            for q in range(1, self.w - 1):
                s = (s + self.hist[:, q]).astype(np.float32)
            if self.w > 1:
                s = (s + col).astype(np.float32)
                self.hist = np.concatenate([self.hist[:, 1:], col[:, None]], axis=1)
            avg = (s / np.float32(self.w)).astype(np.float32)
            f = (g["seen"] + 1 >= self.w) & (avg.astype(np.float64) > self.cutoff)
            g["seen"] += 1
            g["flags"] = (g["flags"] << np.uint64(1)) | f.astype(np.uint64)
            rows = np.nonzero(g["armed"] >= 0)[0]
            if rows.size:
                reason = self._segment(rows, f[rows], p)
                done = reason != 0
                if done.any():
                    self._end(rows[done], reason[done], p)
            self.positions.append(p)
            self.steps += 1

    def flags(self):
        """each row's flag of every step, newest in bit 0 (the uint64 the state keeps)"""
        return self.rows["flags"].copy()

    def arm(self, ids):
        """global ids, in order; ids outside the set ignored, a row taken once per call"""
        taken = set()
        L = min(self.lookback, self.steps)
        for i in ids:
            i = int(i)
            if not 0 <= i < self.n_streams or self.row_of[i] < 0 or self.row_of[i] in taken:
                continue
            r = int(self.row_of[i])
            taken.add(r)
            one = np.array([r])
            self._fresh(one)
            self.rows["armed"][r] = i
            fl = int(self.rows["flags"][r])
            for k in range(L - 1, -1, -1):
                p = self.positions[self.steps - 1 - k]
                reason = self._segment(one, np.array([bool((fl >> k) & 1)]), p)
                if reason[0]:
                    self._end(one, reason, p)
                    break

    def disarm(self, ids):
        for i in ids:
            if 0 <= int(i) < self.n_streams and self.row_of[int(i)] >= 0:
                r = int(self.row_of[int(i)])
                self.rows["armed"][r] = -1
                self._fresh(np.array([r]))

    def reset(self, ids=None, counters=None):
        rows = range(self.members.size) if ids is None else [int(self.row_of[int(i)]) for i in ids
                                                             if 0 <= int(i) < self.n_streams and self.row_of[int(i)] >= 0]
        rows = np.asarray(list(rows), np.int64)
        self.rows["armed"][rows] = -1
        self._fresh(rows)
        self.hist[rows] = 0
        self.rows["seen"][rows] = 0
        self.rows["flags"][rows] = 0
        if ids is None:                               # a whole reset: a new baseline, and no replay reaches across it
            self.base = tuple(counters)
            self.steps, self.positions = 0, []

    def drain(self):
        ev = np.array(self.events, EVENT) if self.events else np.zeros(0, EVENT)
        n = self.count
        self.events, self.count = [], 0
        return ev, n

    def armed_ids(self):
        return self.rows["armed"].astype(np.int32)

    def ended_ids(self):
        out = np.full(self.capacity, -1, np.int32)
        out[:len(self.events)] = [e[0] for e in self.events]
        return out

    def positions64(self):
        out = np.zeros(64, np.int64)
        last = self.positions[::-1][:64]
        out[:len(last)] = last
        return out

    def state(self):
        d = {"hist": self.hist.copy()}
        d.update({k: self.rows[k].astype(np.uint64 if k == "flags" else (np.int64 if k in ("seen", "start_sample", "speech_end_sample") else np.int32))
                  for k in ROW_FIELDS})
        d.update(samples_seen=self.base[0], buffered=self.base[1], pending=self.base[2], steps=self.steps, positions=self.positions64())
        return d


def command_span(e, pre, post, max_samples):
    """(a, length) of one event's command"""
    end = e["end_sample"]
    if e["reason"] == END_OF_SPEECH:
        end = min(e["speech_end_sample"] + post, end)
    a = int(e["start_sample"]) - pre
    return a, int(max(0, min(end - a, max_samples)))


def commands(events, count, capacity, pre, post, max_samples, seen, C, last_C):
    """clips [capacity, max_samples] and lengths [capacity] from last_C(stream) -> the stream's last C history samples (the
    positions [seen - C, seen)), in slot order"""
    clips = np.zeros((capacity, max_samples), np.int16)
    lengths = np.zeros(capacity, np.int32)
    for i in range(min(count, capacity)):
        a, n = command_span(events[i], pre, post, max_samples)
        lengths[i] = n
        ring = last_C(int(events[i]["stream"]))
        t = a + np.arange(n)
        ok = (t >= seen - C) & (t < seen)
        clips[i, :n][ok] = ring[t[ok] - (seen - C)]
    return clips, lengths
