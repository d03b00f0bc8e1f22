"""Per-row cutoffs in both streaming detectors (mww_set_detector_cutoffs, mww_set_multi_detector_cutoffs; StreamDetector and
MultiModelDetector.set_cutoffs), the parts that need no GPU: the NumPy reference (tests/detector_cutoffs_ref.py) against the
uniform references when every cutoff is equal and against the offline rule per row at that row's cutoff; the per-row bodies
of microwakeword_b200/csrc/mww_detector.h (both forms) and mww_detector_models.h built for the host
(tests/emul_detector_cutoffs.cc) against that reference bit for bit, with averages equal to a cutoff, NaN, windows 1 and 32,
every split into calls, cutoff changes between calls, a VAD with per-row cutoffs and resets; the new symbols, the new
library's kernels and the old kernels' instruction hashes; argument checks that need no detector; the loud failure without a
GPU."""

import ctypes
import hashlib
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from detector_cutoffs_ref import ModelsRowsRef, RowsRef
from detector_models_ref import MEVENT, OFF, VAD, WAKE, ModelsRef, call_steps, same_model_events, same_model_state
from detector_ref import EVENT, DetectorRef, same_events, same_state

from oracle import detection_ref as D

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(ROOT, "microwakeword_b200", "csrc")
_BUILD = tempfile.TemporaryDirectory(prefix="mww_detector_cutoffs_test_")
_emul = None


def emul():
    global _emul
    if _emul is None:
        so = os.path.join(_BUILD.name, "libemul_detector_cutoffs.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "emul_detector_cutoffs.cc")], check=True)
        _emul = ctypes.CDLL(so)
        vp, i32, ll = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong
        for fn in (_emul.emul_rows_update_thread, _emul.emul_rows_update_warp):
            fn.restype = ll
            fn.argtypes = [i32, i32, vp, vp, vp, vp, vp, i32, i32, ll, vp, i32]
        model_args = [i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]
        _emul.emul_rows_models_update.restype = ll
        _emul.emul_rows_models_update.argtypes = model_args + [vp, vp, vp, vp, vp, vp, i32]
        _emul.emul_rows_models_reset.restype = None
        _emul.emul_rows_models_reset.argtypes = model_args + [vp, i32]
    return _emul


def _i32(v):
    return np.ascontiguousarray(v, np.int32)


def _ptrs(arrays):
    return (ctypes.c_void_p * len(arrays))(*[None if a is None else a.ctypes.data for a in arrays])


class EmulRows:
    """the per-row plain body on host state, `form` = "thread" or "warp"; the interface of RowsRef"""

    def __init__(self, form, n_rows, cutoff, window=5, cooldown_slices=25):
        self.fn = getattr(emul(), "emul_rows_update_" + form)
        self.n_rows, self.window, self.cooldown_slices = n_rows, window, cooldown_slices
        self.cut = np.full(n_rows, cutoff, np.float64)
        self.hist = np.zeros((n_rows, window - 1), np.float32)
        self.seen = np.zeros(n_rows, np.int64)
        self.cooldown = np.full(n_rows, cooldown_slices, np.int32)

    def set_cutoffs(self, rows, cutoffs):
        rows = np.asarray(rows, np.int64).reshape(-1)
        self.cut[rows] = np.broadcast_to(np.asarray(cutoffs, np.float64), rows.shape)

    def reset(self, rows=None):
        rows = slice(None) if rows is None else [r for r in np.asarray(rows).reshape(-1) if 0 <= r < self.n_rows]
        self.hist[rows] = 0
        self.seen[rows] = 0
        self.cooldown[rows] = self.cooldown_slices

    def update(self, probs):
        probs = np.ascontiguousarray(probs, np.float32).reshape(self.n_rows, -1)
        n = probs.shape[1]
        cap = self.n_rows * max(n, 1)
        buf = np.zeros(cap, [("stream", np.int32), ("reserved", np.int32), ("step", np.int64), ("score", np.float32), ("pad", np.int32)])
        got = self.fn(self.window, self.cooldown_slices, self.cut.ctypes.data, self.hist.ctypes.data, self.seen.ctypes.data,
                      self.cooldown.ctypes.data, probs.ctypes.data, self.n_rows, n, n, buf.ctypes.data, cap)
        ev = np.zeros(got, EVENT)
        ev["stream"], ev["step"], ev["score"] = buf["stream"][:got], buf["step"][:got], buf["score"][:got]
        return ev

    def state(self):
        return dict(hist=self.hist.copy(), seen=self.seen.copy(), cooldown=self.cooldown.copy())


class EmulModelsRows:
    """the per-row models body on host state in the device layout; the interface of ModelsRowsRef"""

    def __init__(self, n_streams, roles, windows, cutoffs, cooldowns, strides, streams=None):
        K = len(roles)
        self.n_streams, self.K, self.roles = n_streams, K, list(roles)
        self.windows = [int(w) for w in windows]
        self.streams = [np.arange(n_streams, dtype=np.int32) if streams is None or streams[k] is None else _i32(streams[k]) for k in range(K)]
        self.inv, self.lookup = [], []
        for s in self.streams:
            inv = np.full(n_streams, -1, np.int32)
            inv[s] = np.arange(s.size)
            self.lookup.append(inv)
            self.inv.append(None if s.size == n_streams else inv)
        self.hist = [np.zeros((max(w - 1, 1), max(s.size, 1)), np.float32) for w, s in zip(self.windows, self.streams)]
        self.seen = [np.zeros(max(s.size, 1), np.int64) for s in self.streams]
        self.flag = [np.zeros(max(s.size, 1), np.int32) for s in self.streams]
        self.cut = [np.full(max(s.size, 1), c, np.float64) for s, c in zip(self.streams, cutoffs)]
        self.arrays = (_i32(roles), _i32(windows), _i32(cooldowns), np.ascontiguousarray(cutoffs, np.float64), _i32(strides),
                       _i32([s.size for s in self.streams]))
        self.reset()

    def set_cutoffs(self, k, stream_ids, cutoffs):
        ids = np.asarray(stream_ids, np.int64).reshape(-1)
        self.cut[k][self.lookup[k][ids]] = np.broadcast_to(np.asarray(cutoffs, np.float64), ids.shape)

    def _model_args(self):
        r, w, c, cut, s, n = self.arrays
        return [self.n_streams, self.K, r.ctypes.data, w.ctypes.data, c.ctypes.data, cut.ctypes.data, _ptrs(self.cut), s.ctypes.data,
                n.ctypes.data, _ptrs(self.inv), _ptrs(self.hist), _ptrs(self.seen), _ptrs(self.flag)]

    def reset(self, ids=None):
        a = None if ids is None else _i32(np.asarray(ids).reshape(-1))
        emul().emul_rows_models_reset(*self._model_args(), None if a is None else a.ctypes.data, 0 if a is None else a.size)

    def update(self, probs, n_steps, pending):
        keep = []
        for k in range(self.K):
            if probs[k] is None or self.roles[k] == OFF or probs[k].size == 0:
                keep.append(np.zeros((1, 1), np.float32))
                continue
            keep.append(np.ascontiguousarray(probs[k], np.float32))
        pitch = np.asarray([k.shape[1] for k in keep], np.int64)
        cap = max(1, self.n_streams * max(n_steps) * self.K)
        buf = np.zeros(cap, [("stream", np.int32), ("reserved", np.int32), ("step", np.int64), ("score", np.float32), ("pad", np.int32)])
        fired = np.full(cap, -1, np.int32)
        n, p = _i32(n_steps), _i32(pending)
        got = emul().emul_rows_models_update(*self._model_args(), _ptrs(keep), pitch.ctypes.data, n.ctypes.data, p.ctypes.data,
                                             buf.ctypes.data, fired.ctypes.data, cap)
        assert got >= 0
        ev = np.zeros(got, MEVENT)
        ev["stream"], ev["model"], ev["step"], ev["score"] = buf["stream"][:got], buf["reserved"][:got], buf["step"][:got], buf["score"][:got]
        return ev

    def state(self):
        out = []
        for k in range(self.K):
            if self.roles[k] == OFF:
                out.append(None)
                continue
            n, w = self.streams[k].size, self.windows[k]
            out.append({"hist": np.ascontiguousarray(self.hist[k][:w - 1, :n].T), "seen": self.seen[k][:n].copy(),
                        ("active" if self.roles[k] == VAD else "cooldown"): self.flag[k][:n].copy()})
        return out


# ---- cases ------------------------------------------------------------------------------------------------------------------
def splits(total, rng, count=8):
    """call-size sequences summing to `total`: one call, single steps, and seeded mixtures with empty calls"""
    out = [[total], [1] * total]
    for _ in range(count):
        seq, left = [], total
        while left:
            s = min(int(rng.choice([0, 1, 2, 3, 7, 33, 64])), left)
            seq.append(s)
            left -= s
        out.append(seq)
    return out


def _probs(rng, R, T):
    p = rng.random((R, T)).astype(np.float32)
    p[1] = 0.99                                          # fires as often as the cooldown allows
    p[2, T // 3:T // 3 + 4] = np.nan                     # never fires while the NaN is in the window
    p[3] = np.float32(0.5)                               # every average is exactly 0.5
    p[4:6] = np.float32(0.75)
    return p


def _row_cutoffs(rng, R, base):
    """random per-row cutoffs, including cutoffs equal to the row's averages (rows 3 and 4: no event) and one ulp below
    them (row 5 against constant 0.75: fires)"""
    c = np.round(rng.uniform(0.3, 0.9, R), 2)
    c[0] = base
    c[3], c[4] = 0.5, 0.75
    c[5] = float(np.nextafter(np.float32(0.75), np.float32(0)))
    return c


def _run(det, probs, seq, changes=None):
    """feed `probs` to `det` in calls of the sizes `seq`; changes: {call index: (rows, cutoffs)} applied before that call"""
    evs, at = [], 0
    for c, n in enumerate(seq):
        if changes and c in changes:
            det.set_cutoffs(*changes[c])
        evs.append(det.update(probs[:, at:at + n]))
        at += n
    return np.concatenate(evs) if evs else np.zeros(0, EVENT)


# ---- the reference ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("window,cooldown", [(1, 0), (5, 25), (32, 3)])
def test_reference_with_equal_cutoffs_is_the_uniform_reference(window, cooldown):
    rng = np.random.default_rng(window + cooldown)
    probs = _probs(rng, 9, 150)
    plain = DetectorRef(9, 0.5, window, cooldown)
    want = plain.update(probs)
    for per_row in (False, True):
        ref = RowsRef(9, 0.5, window, cooldown)
        if per_row:
            ref.set_cutoffs(range(9), 0.5)
        assert same_events(ref.update(probs), want) and same_state(ref.state(), plain.state())


@pytest.mark.parametrize("window,cooldown", [(1, 0), (5, 25), (32, 75)])
def test_reference_rows_are_the_offline_rule_at_their_cutoffs(window, cooldown):
    """the rule mww_false_accept_counts runs, per row at that row's cutoff (oracle/detection_ref.py, pinned to the
    reference's own counts through tests/golden/detection_golden.npz in tests/test_detector.py)"""
    g = np.load(os.path.join(GOLDEN, "detection_golden.npz"))
    rng = np.random.default_rng(window)
    R = 16
    tracks = rng.random((R, 333)).astype(np.float32)
    levels = np.asarray(g["cutoffs"], np.float64)                 # the 101 cutoffs of the reference's ROC
    cut = rng.choice(levels[(levels >= 0.3) & (levels <= 0.8)], R)
    ref = RowsRef(R, 0.5, window, cooldown)
    ref.set_cutoffs(np.arange(R), cut)
    ev = ref.update(tracks)
    assert ev.size > 0
    for r in range(R):
        avg = D.moving_average(tracks[r], window)
        mine = ev[ev["stream"] == r]
        assert mine.size == D.false_accept_counts(avg, [cut[r]], cooldown)[0], r
        assert np.array_equal(mine["score"], avg[mine["step"] - (window - 1)])


def test_models_reference_with_equal_cutoffs_is_the_uniform_one_and_without_a_vad_per_row_plain_detectors():
    rng = np.random.default_rng(4)
    S, strides, windows, cooldowns, cut = 40, [3, 5, 3], [5, 2, 3], [10, 0, 0], [0.55, 0.6, 0.5]
    streams = [None, np.flatnonzero(rng.random(S) < 0.6).astype(np.int32), np.arange(5, S, dtype=np.int32)]
    seqs = [rng.random((S if s is None else s.size, 80 // st + 1)).astype(np.float32) for s, st in zip(streams, strides)]
    for roles in ([WAKE, WAKE, VAD], [WAKE, WAKE, OFF]):
        uni, rows = ModelsRef(S, roles, windows, cut, cooldowns, strides, streams), ModelsRowsRef(S, roles, windows, cut, cooldowns, strides, streams)
        for k in (0, 1) + ((2,) if roles[2] == VAD else ()):
            rows.set_cutoffs(k, rows.streams[k], cut[k])
        want = _feed_models(uni, seqs, strides, [0, 0, 0], [80])
        assert same_model_events(_feed_models(rows, seqs, strides, [0, 0, 0], [80]), want)
        assert same_model_state(rows.state(), uni.state())
    # without a VAD, per-row cutoffs: model k is a per-row plain detector over its set
    roles = [WAKE, WAKE, OFF]
    rows = ModelsRowsRef(S, roles, windows, cut, cooldowns, strides, streams)
    c = [rng.uniform(0.3, 0.8, rows.streams[k].size) for k in range(2)]
    for k in (0, 1):
        rows.set_cutoffs(k, rows.streams[k], c[k])
    got = _feed_models(rows, seqs, strides, [0, 0, 0], [80])
    for k in (0, 1):
        plain = RowsRef(rows.streams[k].size, 0.5, windows[k], cooldowns[k], stream_ids=rows.streams[k])
        plain.set_cutoffs(np.arange(rows.streams[k].size), c[k])
        want = plain.update(seqs[k][:, :80 // strides[k]])
        assert same_events(got[got["model"] == k], want)


def _feed_models(det, seqs, strides, pending0, row_calls, changes=None, resets=None):
    pending, at, evs = list(pending0), [0] * len(strides), []
    for c, rows in enumerate(row_calls):
        for k, ids, v in (changes or {}).get(c, []):
            det.set_cutoffs(k, ids, v)
        if resets and c in resets:
            det.reset(resets[c])
        n, after = call_steps(strides, pending, rows)
        probs = [None if s is None else s[:, a:a + m] for s, a, m in zip(seqs, at, n)]
        evs.append(det.update(probs, n, pending))
        at, pending = [a + m for a, m in zip(at, n)], after
    return np.concatenate(evs) if evs else np.zeros(0, MEVENT)


# ---- the header's per-row bodies against the reference -------------------------------------------------------------------------
@pytest.mark.parametrize("window,cooldown", [(1, 0), (1, 3), (5, 25), (7, 2), (32, 0), (32, 25)])
def test_plain_forms_equal_the_reference_for_every_split_and_cutoff_change(window, cooldown):
    rng = np.random.default_rng(10 * window + cooldown)
    R, T = 12, 140
    probs = _probs(rng, R, T)
    cut = _row_cutoffs(rng, R, 0.5)
    for i, seq in enumerate(splits(T, rng)):
        # cutoff changes between calls (some rows, scalar and per-row values), and a reset that must keep the cutoffs
        mid = len(seq) // 2
        changes = {mid: ([0, 6, 7], [0.95, 0.2, float(cut[7])]), mid + 1: ([8], 0.1)} if i % 2 else None
        ref = RowsRef(R, 0.5, window, cooldown)
        ref.set_cutoffs(np.arange(R), cut)
        want, at = [], 0
        forms = [EmulRows(f, R, 0.5, window, cooldown) for f in ("thread", "warp")]
        for f in forms:
            f.set_cutoffs(np.arange(R), cut)
        got = [[], []]
        for c, n in enumerate(seq):
            if changes and c in changes:
                for d in [ref] + forms:
                    d.set_cutoffs(*changes[c])
            if i % 3 == 2 and c == mid:
                for d in [ref] + forms:
                    d.reset([1, 3, 40])
            want.append(ref.update(probs[:, at:at + n]))
            for g, f in zip(got, forms):
                g.append(f.update(probs[:, at:at + n]))
            at += n
        want = np.concatenate(want)
        assert not (want["stream"] == 3).any() and not (want["stream"] == 4).any() and (want["stream"] == 5).any()
        for g, f in zip(got, forms):
            assert same_events(np.concatenate(g), want), (seq, f.fn)
            assert same_state(f.state(), ref.state())


def test_row_of_a_per_row_detector_is_a_uniform_detector_at_its_cutoff():
    rng = np.random.default_rng(3)
    R, T, window, cooldown = 10, 120, 5, 4
    probs = _probs(rng, R, T)
    cut = _row_cutoffs(rng, R, 0.6)
    for form in ("thread", "warp"):
        det = EmulRows(form, R, 0.5, window, cooldown)
        det.set_cutoffs(np.arange(R), cut)
        got = _run(det, probs, [3, 50, 1, 66])
        for r in range(R):
            one = DetectorRef(R, cut[r], window, cooldown)
            want = one.update(probs)
            assert same_events(got[got["stream"] == r], want[want["stream"] == r]), (form, r)
            assert all(np.array_equal(det.state()[k][r], one.state()[k][r]) for k in ("hist", "seen", "cooldown"))


def _models_case(seed, windows, S=45):
    rng = np.random.default_rng(seed)
    roles = [WAKE, VAD, WAKE]
    strides = [3, int(rng.integers(2, 9)), 3]
    cooldowns = [int(rng.choice([0, 3, 25])), 0, int(rng.choice([0, 1, 10]))]
    cut = [0.6, 0.5, 0.55]
    streams = [None, np.flatnonzero(rng.random(S) < 0.8).astype(np.int32), np.flatnonzero(rng.random(S) < 0.5).astype(np.int32)]
    total = 240
    pending0 = [int(rng.integers(0, s)) for s in strides]
    seqs = []
    for k in range(3):
        rows = S if streams[k] is None else streams[k].size
        n = (pending0[k] + total) // strides[k]
        if roles[k] == VAD:
            runs = (rng.random((rows, n // 4 + 2)) < 0.6).astype(np.float32)
            p = (np.repeat(runs, 4, 1)[:, :n] * 0.9 + 0.05 * rng.random((rows, n))).astype(np.float32)
            p[0, n // 2] = np.nan
        else:
            p = rng.random((rows, n)).astype(np.float32)
            p[1] = np.float32(0.5)                               # averages exactly 0.5
            p[2, 10:14] = np.nan
        seqs.append(p)
    ids = [np.arange(S, dtype=np.int32) if s is None else s for s in streams]
    row_cut = [np.round(rng.uniform(0.3, 0.8, i.size), 2) for i in ids]
    row_cut[0][1] = 0.5                                          # equal to every average of that row
    return dict(S=S, roles=roles, windows=windows, cooldowns=cooldowns, cut=cut, strides=strides, streams=streams, ids=ids,
                row_cut=row_cut, pending0=pending0, total=total, seqs=seqs, rng=rng)


@pytest.mark.parametrize("seed,windows", [(1, [5, 3, 5]), (2, [1, 1, 32]), (3, [32, 5, 1]), (4, [5, 9, 2])])
def test_models_body_equals_the_reference_for_every_split_with_vad_changes_and_resets(seed, windows):
    c = _models_case(seed, windows)
    rng = c["rng"]
    args = (c["S"], c["roles"], c["windows"], c["cut"], c["cooldowns"], c["strides"], c["streams"])
    row_splits = [[c["total"]], [3] * (c["total"] // 3)]
    for _ in range(5):
        seq, left = [], c["total"]
        while left:
            s = min(int(rng.choice([0, 1, 2, 3, 5, 16, 40])), left)
            seq.append(s)
            left -= s
        row_splits.append(seq)
    for i, seq in enumerate(row_splits):
        first = [(k, c["ids"][k], c["row_cut"][k]) for k in range(3)]
        mid = len(seq) // 2
        changes = {0: first}
        if i % 2:
            changes[mid] = [(0, c["ids"][0][:5], 0.97), (1, c["ids"][1][3:9], 0.2), (2, c["ids"][2][-1:], 0.1)]
        resets = {mid + 1: [0, 5, 7, c["S"] + 2]} if i % 3 == 1 else None
        ref, em = ModelsRowsRef(*args), EmulModelsRows(*args)
        want = _feed_models(ref, c["seqs"], c["strides"], c["pending0"], seq, changes, resets)
        got = _feed_models(em, c["seqs"], c["strides"], c["pending0"], seq, changes, resets)
        assert want.size > 0
        assert same_model_events(got, want), (seed, seq)
        assert same_model_state(em.state(), ref.state())
        for k in range(3):
            assert np.array_equal(em.cut[k][:c["ids"][k].size], ref.get_cutoffs(k))
        if i == 0:      # the row whose averages all equal its cutoff never fires
            assert not ((want["model"] == 0) & (want["stream"] == 1)).any()


def test_models_body_with_equal_cutoffs_is_the_uniform_body():
    """the per-row body over descriptors holding the model's cutoff in every row against the uniform reference"""
    c = _models_case(9, [5, 3, 5])
    args = (c["S"], c["roles"], c["windows"], c["cut"], c["cooldowns"], c["strides"], c["streams"])
    em = EmulModelsRows(*args)
    want = _feed_models(ModelsRef(*args), c["seqs"], c["strides"], c["pending0"], [c["total"]])
    assert same_model_events(_feed_models(em, c["seqs"], c["strides"], c["pending0"], [c["total"]]), want)


# ---- build and ABI ---------------------------------------------------------------------------------------------------------------
NEW = ("mww_set_detector_cutoffs", "mww_get_detector_cutoffs", "mww_set_multi_detector_cutoffs", "mww_get_multi_detector_cutoffs")


def test_new_symbols_are_declared_and_exported():
    from microwakeword_b200 import _lib, build
    L = _lib.lib()
    assert all(n in _lib.EXPORTS and hasattr(L, n) for n in NEW)
    syms = subprocess.run(["nm", "-D", "--defined-only", build.OUT], capture_output=True, text=True, check=True).stdout
    assert all(re.search(r"\bT %s\b" % n, syms) for n in NEW)
    hdr = re.sub(r"\s*\n\s*\*\s*", " ", open(os.path.join(ROOT, "include", "mww.h")).read())
    for line in ("(double)avg > c_r in place of (double)avg > cutoff", "Per-row mode with every c_r = c is bit-identical to uniform mode",
                 "mww_false_accept_counts at c_r", "Ordered on cu_stream", "resets keep the cutoffs", "n == 0 does nothing and does not switch mode"):
        assert line in hdr, line


def _cuobjdump():
    from microwakeword_b200 import _lib, build
    tool = os.path.join(os.path.dirname(build.NVCC), "cuobjdump")
    if not os.path.exists(tool):
        pytest.skip("cuobjdump is not installed next to nvcc")
    _lib.lib()
    return tool


def _sass_hashes(so):
    text = subprocess.run([_cuobjdump(), "-sass", so], capture_output=True, text=True, check=True).stdout
    words, name = {}, None
    for line in text.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1)
            words[name] = []
        elif name:
            words[name] += re.findall(r"/\* (0x[0-9a-f]{16}) \*/", line)
    return {n: hashlib.sha256(" ".join(w).encode()).hexdigest() for n, w in words.items()}


def test_uniform_detector_kernels_keep_their_instructions():
    """libmww_detector.so and libmww_detector_models.so: the same kernels, instruction for instruction, as before per-row
    cutoffs (their names now carry the row-cutoff template argument)"""
    from microwakeword_b200 import build
    before = json.load(open(os.path.join(GOLDEN, "sass_kernels_before_detector_cutoffs.json")))
    keys = {"libmww_detector.so": [("update_thread", r"detector_update_kernelILb0ELb0E"), ("update_warp", r"detector_update_kernelILb1ELb0E"),
                                   ("reset", r"detector_reset_kernel")],
            "libmww_detector_models.so": [("models_update", r"detector_models_update_kernelINS_11DetectModelE"),
                                          ("models_reset", r"detector_models_reset_kernel")]}
    for lib, out in ((build.DET_OUT, "libmww_detector.so"), (build.MD_OUT, "libmww_detector_models.so")):
        got = _sass_hashes(lib)
        assert len(got) == len(keys[out]), got
        for key, pat in keys[out]:
            (h,) = [h for n, h in got.items() if re.search(pat, n)]
            assert h == before[out][key], (out, key)


def test_cutoffs_library_holds_exactly_its_kernels_without_spills():
    from microwakeword_b200 import build
    assert os.path.basename(build.DC_OUT) == "libmww_detector_cutoffs.so" and build.DC_SOURCES == ["mww_detector_cutoffs.cu"]
    res = subprocess.run([_cuobjdump(), "-res-usage", build.DC_OUT], capture_output=True, text=True, check=True).stdout
    found = re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", res)
    names = sorted(n for n, *_ in found)
    assert len(names) == 3, res[-2000:]
    assert sum(bool(re.search(r"detector_update_kernelILb[01]ELb1E", n)) for n in names) == 2
    assert sum("detector_models_update_kernelINS_15DetectModelRowsE" in n for n in names) == 1
    assert all(int(stack) == int(local) == 0 for _, _, stack, local in found), found
    flags = [f for f in build.FLAGS if f not in ("-shared", "-cudart", "static")]
    rep = subprocess.run([build.NVCC] + flags + ["-cubin", "-Xptxas", "-v", "-o", os.path.join(_BUILD.name, "cutoffs.cubin"),
                                                 os.path.join(CSRC, "mww_detector_cutoffs.cu")], capture_output=True, text=True, check=True).stderr
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", rep)
    assert len(spills) == 3 and all(int(a) == int(b) == 0 for a, b in spills), rep
    if shutil.which("readelf"):
        dyn = subprocess.run(["readelf", "-d", build.OUT], capture_output=True, text=True, check=True).stdout
        assert "[libmww_detector_cutoffs.so]" in dyn and "$ORIGIN" in dyn


# ---- refusals that need no detector, and the loud failure without a GPU ----------------------------------------------------------
def test_null_detector_and_bad_lists_are_refused():
    from microwakeword_b200 import _lib
    from microwakeword_b200.detection import _cutoff_list
    L = _lib.lib()
    rows, cut = (ctypes.c_int32 * 1)(0), (ctypes.c_double * 1)(0.5)
    assert L.mww_set_detector_cutoffs(None, rows, cut, 1, None) == -1 and b"NULL" in L.mww_last_error(None)
    assert L.mww_get_detector_cutoffs(None, cut) == -1
    assert L.mww_set_multi_detector_cutoffs(None, 0, rows, cut, 1, None) == -1
    assert L.mww_get_multi_detector_cutoffs(None, 0, cut) == -1
    for ids, c in (([[0, 1]], 0.5), ([0.5], 0.5), ([True], 0.5), ([0, 1], [0.5, 0.6, 0.7]), ([0], float("nan")), ([0, 1], [0.5, np.inf]),
                   ([0], "0.5"), ([0], 0.5 + 1j), ([2 ** 40], 0.5)):
        with pytest.raises(ValueError):
            _cutoff_list(ids, c, "rows")
    i, c = _cutoff_list(np.asarray([3, 1], np.int64), 0.25, "rows")
    assert i.dtype == np.int32 and c.dtype == np.float64 and c.tolist() == [0.25, 0.25]
    assert _cutoff_list([], 0.5, "rows")[0].size == 0


def test_no_cpu_fallback_without_a_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present; the loud-failure path is exercised on GPU-less hosts")
    from microwakeword_b200 import _lib
    from microwakeword_b200.detection import StreamDetector
    with pytest.raises(_lib.MwwError) as e:
        StreamDetector(8, cutoff=0.5)
    assert e.value.code == -3 and "no CUDA device" in str(e.value)
    tool = os.path.join(ROOT, "tools", "detector_cutoffs_time.py")
    res = subprocess.run([sys.executable, tool, "--rows", "64"], capture_output=True, text=True)
    assert res.returncode != 0 and "CUDA" in res.stderr
