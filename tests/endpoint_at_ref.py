"""tests/endpoint_at_ref.py -- TEST INFRASTRUCTURE: the positioned arm of the endpointer (mww_endpointer_arm_at, include/mww.h
"positioned arm") in NumPy, written from the rule text on top of endpoint_ref.EndpointRef.  Each row also keeps a mute count
and a `placed` bit (start_sample fixed by arm_at, no step taken since); the segmenter step mutes, and every path to fresh
segmenter state clears both."""

import numpy as np

import endpoint_ref as R

PLACED = 1 << 30


class EndpointAtRef(R.EndpointRef):
    def __init__(self, *args, **kw):
        super().__init__(*args, **kw)
        n = self.members.size
        self.mute = np.zeros(n, np.int64)
        self.placed = np.zeros(n, bool)

    def q(self):
        """the position of the newest step consumed (where it would have been, with none since a whole reset)"""
        S, buffered, pending = self.base
        return R.position(S, buffered, self.hop, pending, self.stride, 1, 0)

    def _fresh(self, rows):
        super()._fresh(rows)
        self.mute[rows] = 0
        self.placed[rows] = False

    def _segment(self, rows, f, p):
        """one step of the listed armed rows: a row with mute > 0 takes flag 0 and counts it down; a placed row keeps its
        start_sample; otherwise the plain rule"""
        rows = np.asarray(rows)
        m = self.mute[rows]
        f = np.asarray(f, bool) & (m == 0)
        self.mute[rows] = np.maximum(m - 1, 0)
        g = self.rows
        first = rows[(g["elapsed"][rows] == 0) & ~self.placed[rows]]
        g["start_sample"][first] = g["speech_end_sample"][first] = p - self.stride * self.hop
        self.placed[rows] = False
        g["elapsed"][rows] += 1
        on, off = rows[f], rows[~f]
        g["run"][on] += 1
        g["silence"][on] = 0
        g["heard"][on[g["run"][on] >= self.speech_steps]] = 1
        g["speech_end_sample"][on[g["heard"][on] == 1]] = p
        g["run"][off] = 0
        g["silence"][off] += 1
        heard = g["heard"][rows] == 1
        return np.where(heard & (g["silence"][rows] >= self.silence_steps), R.END_OF_SPEECH,
                        np.where(~heard & (g["elapsed"][rows] >= self.timeout_steps), R.NO_SPEECH,
                                 np.where(g["elapsed"][rows] >= self.max_steps, R.MAX_LENGTH, 0)))

    def arm_at(self, ids, positions, skip):
        q, step = self.q(), self.stride * self.hop
        latest = {}                                            # row -> (P', id), the latest position of each row listed
        for i, P in zip(ids, positions):
            i = int(i)
            if not 0 <= i < self.n_streams or self.row_of[i] < 0:
                continue
            r = int(self.row_of[i])
            Pc = min(int(P), q)
            if r not in latest or Pc > latest[r][0]:
                latest[r] = (Pc, i)
        L = min(self.lookback, self.steps)
        g = self.rows
        for r, (Pc, i) in latest.items():
            one = np.array([r])
            self._fresh(one)
            g["armed"][r] = i
            g["start_sample"][r] = g["speech_end_sample"][r] = Pc
            self.placed[r] = True
            fl = int(g["flags"][r])
            ended = False
            for k in range(L - 1, -1, -1):
                p = self.positions[self.steps - 1 - k]
                if p <= Pc:
                    continue
                reason = self._segment(one, np.array([bool((fl >> k) & 1) and p > Pc + skip]), p)
                if reason[0]:
                    self._end(one, reason, p)
                    ended = True
                    break
            if not ended:
                d = Pc + skip - q
                self.mute[r] = d // step if d > 0 else 0
                self.placed[r] = g["elapsed"][r] == 0

    def mute_words(self):
        return (self.mute | np.where(self.placed, PLACED, 0)).astype(np.int32)

    def state(self):
        d = super().state()
        d["mute"] = self.mute_words()
        return d
