"""The media guard's rule (include/mww.h, "media guard") in NumPy, written from the header's text: fingerprints of feature rows,
the lag-minimum mismatch test, and one check call over slots, the ring and the registered clips."""

import numpy as np

BITS = 39


def fingerprint(F):
    """F [T][40] uint16 -> [T - 1] uint64: bit c of word t - 1 is (F[t][c] - F[t][c+1]) - (F[t-1][c] - F[t-1][c+1]) > 0"""
    F = np.asarray(F, np.int64)
    d = F[:, :BITS] - F[:, 1:BITS + 1]
    bits = (d[1:] - d[:-1]) > 0
    return (bits.astype(np.uint64) << np.arange(BITS, dtype=np.uint64)).sum(axis=1, dtype=np.uint64)


def popcount(x):
    x = np.asarray(x, np.uint64)
    return np.unpackbits(x.view(np.uint8).reshape(-1, 8), axis=1).sum(axis=1) if x.size else np.zeros(0, np.int64)


def matches_at(x, y, l, min_overlap, ber_milli):
    t = np.arange(len(x))
    t = t[(t + l >= 0) & (t + l < len(y))]
    O = t.size
    if O < min_overlap:
        return False
    m = int(popcount(x[t] ^ y[t + l]).sum())
    return m * 1000 <= ber_milli * BITS * O


def match(x, y, lags, min_overlap, ber_milli):
    return any(matches_at(x, y, l, min_overlap, ber_milli) for l in lags)


def detection_lags(max_lag):
    return range(-max_lag, max_lag + 1)


def clip_lags(n_x, n_y, min_overlap):
    return range(-(n_x - min_overlap), n_y - min_overlap + 1)


def same_household(hi, si, hj, sj):
    return hi == hj and (hi >= 0 or si == sj)


class Rule:
    def __init__(self, max_lag, min_overlap, ber_milli, min_matches, ring, window):
        self.max_lag, self.min_overlap, self.ber_milli, self.min_matches = max_lag, min_overlap, ber_milli, min_matches
        self.ring_size, self.window = ring, window
        self.ring = []              # appended entries, oldest first: (fp, stream, household, pos)
        self.clips = []

    def check(self, fps, streams, valid, households, positions, confirmed=None):
        """slots in slot order -> (matches, media, passed) int32 arrays; appends the valid slots to the ring"""
        n = len(streams)
        matches, media, passed = np.full(n, -1, np.int32), np.zeros(n, np.int32), np.zeros(n, np.int32)
        kept = self.ring[-self.ring_size:] if self.ring_size else []
        for i in range(n):
            conf = int(confirmed[i]) if confirmed is not None else int(streams[i])
            if not valid[i]:
                passed[i] = conf
                continue
            cands = [(fps[j], streams[j], households[j], positions[j]) for j in range(n) if j != i and valid[j]] + kept
            c = sum(1 for (y, s, h, p) in cands
                    if not same_household(households[i], streams[i], h, s) and abs(int(p) - int(positions[i])) <= self.window
                    and match(fps[i], y, detection_lags(self.max_lag), self.min_overlap, self.ber_milli))
            clip = any(match(fps[i], y, clip_lags(len(fps[i]), len(y), self.min_overlap), self.min_overlap, self.ber_milli) for y in self.clips)
            matches[i] = c
            media[i] = (1 if clip else 0) | (2 if c >= self.min_matches else 0)
            passed[i] = -1 if media[i] else conf
        self.ring += [(fps[i], streams[i], households[i], positions[i]) for i in range(n) if valid[i]]
        self.ring = self.ring[-self.ring_size:] if self.ring_size else []
        return matches, media, passed
