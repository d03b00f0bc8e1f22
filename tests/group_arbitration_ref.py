"""NumPy statement of group arbitration (include/mww.h, "group arbitration"), written from the header's rule alone.

level() measures one candidate from the Ls + Ln samples that end at its position (zeros where the history holds nothing);
ArbRule is grouped detection's window rule (detector_groups_ref.GroupRule) with the arbitrated order: the highest level, then
the highest score, then the earliest position, then the lowest id (row, or global stream for a models detector)."""

import numpy as np

from detector_groups_ref import GroupRule


def energy(x) -> np.float64:
    """(q - r r / L) / L of one span, each operation a separately rounded double operation"""
    x = np.asarray(x, np.int64)
    L = np.float64(x.size)
    q, r = np.float64(int((x * x).sum())), np.float64(int(x.sum()))
    return (q - r * r / L) / L


def level_of(audio, Ls, Ln) -> np.float32:
    """audio: the Ls + Ln samples that end at the candidate, oldest first (noise, then speech)"""
    audio = np.asarray(audio)
    assert audio.shape == (Ls + Ln,)
    return np.float32((energy(audio[Ln:]) + np.float64(1.0)) / (energy(audio[:Ln]) + np.float64(1.0)))


def read_at(ring, S, stream, P, L):
    """the L samples of `stream` that end at P, by the history's read-at rule: a position outside [S - C, S) is zero"""
    C = ring.shape[1]
    pos = np.arange(P - L, P)
    held = (pos >= S - C) & (pos < S)
    out = np.zeros(L, np.int16)
    out[held] = ring[stream, pos[held] % C]
    return out


def level(ring, S, stream, P, Ls, Ln) -> np.float32:
    return level_of(read_at(ring, S, stream, P, Ls + Ln), Ls, Ln)


def better(c, best):
    if best is None:
        return True
    a = (-float(c["level"]), -float(c["score"]), int(c["sample"]), int(c["id"]))
    b = (-float(best["level"]), -float(best["score"]), int(best["sample"]), int(best["id"]))
    return a < b


class ArbRule(GroupRule):
    """GroupRule whose candidates carry `level` and `id` and merge in the arbitrated order"""

    def update(self, cands, a, E):
        out = []
        for key in sorted(set(self.open) | set(cands), key=repr):
            ak = a[key] if isinstance(a, dict) else a
            Ek = E[key] if isinstance(E, dict) else E
            if key in self.open and ak is not None and ak >= self.open[key][0]:
                self._emit(key, out)
            cs = cands.get(key, [])
            if cs:
                if key not in self.open:
                    self.open[key] = [min(int(c["sample"]) for c in cs) + self.W, None, 0]
                w = self.open[key]
                for c in cs:
                    if better(c, w[1]):
                        w[1] = c
                w[2] += len(cs)
            if key in self.open and Ek >= self.open[key][0]:
                self._emit(key, out)
        return out


def levels_of(audio, Ls, Ln) -> np.ndarray:
    """level_of for every row of an int16 [n, Ls + Ln] array, in the same double operations"""
    x = np.asarray(audio, np.int64)
    s, n = x[:, Ln:], x[:, :Ln]
    return levels_from_sums((s * s).sum(1), s.sum(1), (n * n).sum(1), n.sum(1), Ls, Ln)


def levels_from_sums(q_speech, r_speech, q_noise, r_noise, Ls, Ln) -> np.ndarray:
    """levels_of from each span's exact integer sums (sum x^2, sum x)"""
    e = []
    for q, r, L in ((q_speech, r_speech, Ls), (q_noise, r_noise, Ln)):
        q, r, Lf = np.asarray(q).astype(np.float64), np.asarray(r).astype(np.float64), np.float64(L)
        e.append((q - r * r / Lf) / Lf)
    return ((e[0] + 1.0) / (e[1] + 1.0)).astype(np.float32)
