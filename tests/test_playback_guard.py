"""The playback guard (include/mww.h, "playback guard"), the parts that need no GPU: the header bodies built with g++ from
microwakeword_b200/csrc/mww_playback.h by tests/emul_playback_guard.cc against the NumPy statement of the rule in
tests/playback_guard_ref.py -- seeded write/read/check sequences, and every edge: writes in order, with gaps, overlapping into
the past, fully in the past, ahead of S, longer than C, across the ring's wrap, into a fresh row; the release at w = S - C and
S - C + 1; MWW_ENOMEM; the heard rule at r0 = S - C - 1 / S - C, w - C - 1 / w - C and w - 1 / w; a NaN score and the cutoff
and one ulp above it.  Also the structs, the new symbols and their argument types, the refusals before any device work in C and
in Python, the new library's kernels without stack, local memory or spills, and every pre-existing kernel's instructions
against tests/golden/sass_kernels_before_playback_guard.json (the parent's build)."""

import ctypes
import json
import os
import re
import subprocess
import sys
import tempfile
import types

import numpy as np
import pytest

from conftest import GOLDEN, ROOT

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import playback_guard_ref as ref  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(ROOT, "microwakeword_b200", "csrc")
_BUILD = tempfile.TemporaryDirectory(prefix="mww_playback_test_")
_emul = []
vp, i32, ll, dbl = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_double


def emul():
    if not _emul:
        so = os.path.join(_BUILD.name, "libemul_playback_guard.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "emul_playback_guard.cc")], check=True)
        L = ctypes.CDLL(so)
        L.emul_sizes.argtypes = [ctypes.POINTER(i32), ctypes.POINTER(i32)]
        L.emul_write.argtypes = [vp, vp, i32, vp, i32, ll, i32, i32, i32, vp, vp, vp, vp, vp, vp]
        L.emul_write.restype = i32
        L.emul_read.argtypes = [vp, vp, i32, i32, ll, i32, i32, vp, vp, vp, vp]
        L.emul_read.restype = None
        L.emul_heard.argtypes = [vp, vp, i32, i32, ll, i32, i32, ll, vp, vp, vp]
        L.emul_heard.restype = None
        L.emul_slots_detector.argtypes = [i32, ll, vp, vp, i32, ll, ll, vp, vp]
        L.emul_slots_detector.restype = None
        L.emul_decide.argtypes = [i32, vp, vp, dbl, vp, vp, vp, vp]
        L.emul_decide.restype = None
        _emul.append(L)
    return _emul[0]


def test_struct_sizes_match_the_header():
    from microwakeword_b200 import _lib
    r, d = i32(), i32()
    emul().emul_sizes(ctypes.byref(r), ctypes.byref(d))
    assert (r.value, d.value) == (ctypes.sizeof(_lib.MwwPlaybackRule), ctypes.sizeof(_lib.MwwPlaybackGuardDesc)) == (40, 80)


class Guard:
    """the emulated guard (host mirror, device map, ring) and the NumPy rule side by side"""

    def __init__(self, n_streams, rows, C):
        self.n, self.rows, self.C = n_streams, rows, C
        self.row_of, self.stream_of, self.head = np.full(n_streams, -1, np.int32), np.full(rows, -1, np.int32), np.zeros(rows, np.int64)
        self.dev_row_of, self.dev_head = np.full(n_streams, -1, np.int32), np.zeros(rows, np.int64)
        self.ring = np.zeros((rows, C), np.int16)
        self.ref = ref.Rule(n_streams, rows, C)

    def write(self, ids, starts, x, seen):
        ids, starts = np.ascontiguousarray(ids, np.int32), np.ascontiguousarray(starts, np.int64)
        x = np.ascontiguousarray(x, np.int16).reshape(ids.size, -1)
        before = [a.copy() for a in (self.row_of, self.stream_of, self.head, self.ring, self.dev_row_of, self.dev_head)]
        got = emul().emul_write(ids.ctypes.data, starts.ctypes.data, ids.size, x.ctypes.data, x.shape[1], seen, self.C, self.rows, self.n,
                                self.row_of.ctypes.data, self.stream_of.ctypes.data, self.head.ctypes.data, self.ring.ctypes.data,
                                self.dev_row_of.ctypes.data, self.dev_head.ctypes.data)
        want = self.ref.write(ids, starts, x, seen)
        assert (got < 0) == (want == ref.ENOMEM)
        if got < 0:                                          # refused: nothing written or freed
            for a, b in zip(before, (self.row_of, self.stream_of, self.head, self.ring, self.dev_row_of, self.dev_head)):
                assert np.array_equal(a, b)
        self.agree()
        return got

    def reset(self, ids=None):
        for s in (range(self.n) if ids is None else ids):
            r = self.row_of[s]
            if r >= 0:
                self.stream_of[r] = -1
            self.row_of[s] = self.dev_row_of[s] = -1
        self.ref.reset(ids)

    def agree(self):
        """the mirror equals the device map; the streams holding a row and their heads are the rule's"""
        assert np.array_equal(self.row_of, self.dev_row_of)
        held = {int(s): int(self.head[r]) for s, r in enumerate(self.row_of) if r >= 0}
        assert held == self.ref.head
        assert np.array_equal(self.head[self.row_of[self.row_of >= 0]], self.dev_head[self.row_of[self.row_of >= 0]])

    def read(self, ids, ends, L, min_delay=0):
        ids, ends = np.ascontiguousarray(ids, np.int32), np.ascontiguousarray(ends, np.int64)
        out = np.zeros((ids.size, L), np.int16)
        emul().emul_read(ids.ctypes.data, ends.ctypes.data, ids.size, L, min_delay, self.n, self.C, self.ring.ctypes.data,
                         self.dev_row_of.ctypes.data, self.dev_head.ctypes.data, out.ctypes.data)
        for i, (s, e) in enumerate(zip(ids, ends)):
            want = self.ref.read(int(s), int(e) - min_delay, L) if 0 <= s < self.n else np.zeros(L, np.int16)
            assert np.array_equal(out[i], want), (s, e)
        return out

    def heard(self, ids, ends, L, min_delay, seen):
        ids, ends = np.ascontiguousarray(ids, np.int32), np.ascontiguousarray(ends, np.int64)
        out = np.zeros(ids.size, np.int32)
        emul().emul_heard(ids.ctypes.data, ends.ctypes.data, ids.size, L, min_delay, self.n, self.C, seen, self.dev_row_of.ctypes.data,
                          self.dev_head.ctypes.data, out.ctypes.data)
        want = [self.ref.heard(int(s), int(e) - min_delay - L, seen) for s, e in zip(ids, ends)]
        assert list(out) == [int(w) for w in want]
        return out


def audio(rng, n, L):
    return rng.integers(-32768, 32768, (n, L)).astype(np.int16)


def test_writes_at_every_edge_read_as_the_rule():
    rng = np.random.default_rng(1)
    C = 64
    g = Guard(8, 4, C)
    ends = np.arange(-40, 400)
    every = lambda s: g.read(np.full(ends.size, s, np.int32), ends, 16)   # noqa: E731
    g.write([0], [0], audio(rng, 1, 24), 0)           # a fresh row
    every(0)
    g.write([0], [24], audio(rng, 1, 16), 0)          # in order
    every(0)
    g.write([0], [50], audio(rng, 1, 8), 0)           # with a gap [40, 50)
    every(0)
    g.write([0], [30], audio(rng, 1, 20), 0)          # overlapping into the past
    every(0)
    g.write([0], [-100], audio(rng, 1, 20), 0)        # fully in the past: before the ring
    every(0)
    g.write([0], [10], audio(rng, 1, 8), 0)           # fully in the past, inside the ring
    every(0)
    g.write([0], [500], audio(rng, 1, 8), 0)          # ahead of S, a gap longer than C
    every(0)
    g.write([1], [3], audio(rng, 1, 150), 0)          # n > C into a fresh row
    every(1)
    g.write([1], [157], audio(rng, 1, 45), 0)         # across the ring's wrap (157 mod 64 = 29, 29 + 45 > 64)
    every(1)
    g.write([2], [7], audio(rng, 1, 0), 0)            # nothing: the row only moves its head
    every(2)
    for s in range(4):
        every(s)


def test_release_at_w_equal_s_minus_c_and_not_one_later():
    rng = np.random.default_rng(2)
    C = 32
    for seen, freed in ((100 + C, True), (100 + C - 1, False)):
        g = Guard(4, 2, C)
        g.write([0], [60], audio(rng, 1, 40), 0)      # head 100
        g.write([1], [0], audio(rng, 1, 8), 0)        # head 8, freed at any S >= 40
        assert g.write([2], [200], audio(rng, 1, 8), seen) > 0   # row of stream 1 is freed; stream 0's only at S >= 132
        assert (g.row_of[0] < 0) == freed and g.row_of[1] < 0 and g.row_of[2] >= 0


def test_out_of_rows_is_refused_and_changes_nothing():
    rng = np.random.default_rng(3)
    g = Guard(6, 2, 16)
    g.write([0, 1], [0, 0], audio(rng, 2, 16), 0)
    assert g.write([2], [16], audio(rng, 1, 8), 0) < 0
    assert g.write([0, 2], [16, 16], audio(rng, 2, 8), 0) < 0
    assert g.write([0, 1], [16, 16], audio(rng, 2, 8), 0) > 0      # the rows are kept: no new one is needed
    assert g.write([2], [40], audio(rng, 1, 8), 39) < 0            # heads 24 > S - C = 23: nothing is released
    assert g.write([2], [40], audio(rng, 1, 8), 40) > 0            # heads 24 <= S - C = 24: both rows are released
    assert g.row_of[0] < 0 and g.row_of[1] < 0 and g.row_of[2] == 0
    g.reset([2])
    assert g.write([3, 4], [0, 0], audio(rng, 2, 8), 40) > 0


@pytest.mark.parametrize("seed", range(6))
def test_seeded_write_read_sequences_are_the_rule(seed):
    rng = np.random.default_rng(100 + seed)
    n_streams, rows, C = 12, int(rng.integers(2, 9)), int(rng.choice([16, 40, 96]))
    g = Guard(n_streams, rows, C)
    seen, refused = 0, 0
    for call in range(40):
        k = int(rng.integers(1, 5))
        ids = rng.choice(n_streams, k, replace=False)
        L = int(rng.choice([0, 3, 8, 16, 33, C, C + 9]))
        base = seen + int(rng.integers(-2 * C, 2 * C))
        starts = base + rng.integers(-C, C, k)
        refused += g.write(ids, starts, audio(rng, k, L), seen) < 0
        if rng.random() < 0.15:
            g.reset(list(rng.choice(n_streams, 2, replace=False)) if rng.random() < 0.7 else None)
        seen += int(rng.integers(0, C))
        ids = rng.integers(-1, n_streams + 1, 20)
        ends = seen + rng.integers(-3 * C, C, 20)
        g.read(ids, ends, int(rng.integers(1, C + 1)))
        g.heard(ids, ends, int(rng.integers(1, C // 2)), int(rng.integers(0, 5)), seen)
    assert refused < 40


def test_heard_rule_edges():
    """r0 = S - C - 1 / S - C, w - C - 1 / w - C, w - 1 / w"""
    rng = np.random.default_rng(4)
    C, L = 100, 20
    g = Guard(4, 2, C)
    g.write([0], [1000], audio(rng, 1, 300), 0)       # w = 1300: holds [1200, 1300)
    S = 1250                                          # S - C = 1150 < w - C: the head bounds it
    r0s = [1199, 1200, 1299, 1300]
    out = g.heard([0] * 4, [r + L for r in r0s], L, 0, S)
    assert list(out) == [0, 1, 1, 0]
    S = 1310                                          # S - C = 1210 > w - C: S bounds it
    out = g.heard([0] * 4 + [1, -1, 4], [1209 + L, 1210 + L, 1250 + L, 1299 + L, 1250 + L, 1250 + L, 1250 + L], L, 0, S)
    assert list(out) == [0, 1, 1, 1, 0, 0, 0]
    out = g.heard([0, 0], [1210 + L + 7, 1209 + L + 7], L, 7, S)   # min_delay moves r1
    assert list(out) == [1, 0]


def test_decision_nan_and_the_cutoff_exactly():
    cutoff = 0.5
    up = float(np.nextafter(np.float32(0.5), np.float32(1)))
    heard = np.array([1, 1, 1, 0, 0, 1], np.int32)
    scores = np.array([0.5, up, np.nan, 0.99, np.nan, 0.2], np.float32)
    conf = np.array([3, 4, 5, 6, -1, 8], np.int32)
    out = [np.zeros(6, np.float32), np.zeros(6, np.int32), np.zeros(6, np.int32)]
    emul().emul_decide(6, heard.ctypes.data, scores.ctypes.data, cutoff, conf.ctypes.data, *(o.ctypes.data for o in out))
    want = [ref.decide(bool(h), s, cutoff, int(c)) for h, s, c in zip(heard, scores, conf)]
    assert np.array_equal(out[0], np.array([w[0] for w in want], np.float32), equal_nan=True)
    assert list(out[1]) == [w[1] for w in want] == [0, 1, 0, 0, 0, 0]
    assert list(out[2]) == [w[2] for w in want] == [3, -1, 5, 6, -1, 8]


EVENT = np.dtype([("stream", np.int32), ("reserved", np.int32), ("step", np.int64), ("score", np.float32), ("pad", np.int32)])


def test_detector_slots_take_the_verifier_rule():
    seen, post = 100000, 3200
    ev = np.zeros(6, EVENT)
    ev["stream"] = [10, 11, 12, 13, 14, 15]
    ev["reserved"] = [0, 1, 0, 0, 1, 0]
    pos = np.array([90000, 90000, seen - 1000, 50, 7, 8], np.int64)
    sid, end = np.zeros(6, np.int32), np.zeros(6, np.int64)
    emul().emul_slots_detector(6, 4, ev.ctypes.data, pos.ctypes.data, 0, post, seen, sid.ctypes.data, end.ctypes.data)
    assert list(sid) == [10, -1, 12, 13, -1, -1] and list(end[[0, 2, 3]]) == [93200, seen, 3250]
    emul().emul_slots_detector(6, 100, ev.ctypes.data, pos.ctypes.data, -1, 0, seen, sid.ctypes.data, end.ctypes.data)
    assert list(sid) == [10, 11, 12, 13, 14, 15] and list(end) == list(pos)


# ---- build, ABI and refusals ----------------------------------------------------------------------------------------------------------
NEW = {"mww_playback_guard_create": ("const mww_t *h, const void *model_blob, size_t n_bytes, int slots, int rows, int capacity, "
                                     "const mww_playback_rule *rule, mww_playback_guard_t **out", [vp, vp, ctypes.c_size_t, i32, i32, i32, None, None]),
       "mww_playback_guard_destroy": ("mww_playback_guard_t *g", [vp]),
       "mww_playback_guard_info": ("const mww_playback_guard_t *g, mww_playback_guard_desc *out", [vp, None]),
       "mww_playback_write": ("mww_playback_guard_t *g, const int32_t *h_ids, const long long *h_starts, int n, const int16_t *d_audio, "
                              "int n_samples, long long audio_stride, void *cu_stream", [vp, vp, vp, i32, vp, i32, ll, vp]),
       "mww_playback_read": ("mww_playback_guard_t *g, const int32_t *d_ids, const long long *d_ends, int n, int n_samples, int16_t *d_out, "
                             "long long out_stride, void *cu_stream", [vp, vp, vp, i32, i32, vp, ll, vp]),
       "mww_playback_reset": ("mww_playback_guard_t *g, const int32_t *h_ids, int n, void *cu_stream", [vp, vp, i32, vp]),
       "mww_playback_get_heads": ("const mww_playback_guard_t *g, int32_t *h_rows, int64_t *h_heads", [vp, vp, vp]),
       "mww_playback_check_streams": ("mww_playback_guard_t *g, const int32_t *d_ids, const long long *d_ends, int n, const int32_t *d_confirmed, "
                                      "float *d_scores, int32_t *d_flagged, int32_t *d_passed, void *cu_stream", [vp, vp, vp, i32, vp, vp, vp, vp, vp]),
       "mww_playback_check_detections_at": ("mww_playback_guard_t *g, mww_detector_t *det, int model, long long post, const int32_t *d_confirmed, "
                                            "float *d_scores, int32_t *d_flagged, int32_t *d_passed, void *cu_stream",
                                            [vp, vp, i32, ll, vp, vp, vp, vp, vp])}


def test_new_symbols_are_declared_and_exported_with_their_arguments():
    from microwakeword_b200 import _lib, build
    L = _lib.lib()
    syms = subprocess.run(["nm", "-D", "--defined-only", build.OUT], capture_output=True, text=True, check=True).stdout
    hdr = re.sub(r"\s+", " ", open(os.path.join(ROOT, "include", "mww.h")).read())
    for name, (sig, args) in NEW.items():
        assert name in _lib.EXPORTS and re.search(r"\bT %s\b" % name, syms), name
        assert "int %s(%s);" % (name, sig) in hdr, name
        got = getattr(L, name).argtypes
        assert len(got) == len(args) and all(a is None or g == a for g, a in zip(got, args)), name


def rule(**kw):
    from microwakeword_b200 import _lib
    r = dict(n_samples=24000, window=5, ignore_steps=25, pad=0, min_delay=0, max_delay=4800, cutoff=0.5)
    r.update(kw)
    return _lib.MwwPlaybackRule(*(r[k] for k, _ in _lib.MwwPlaybackRule._fields_))


@pytest.mark.parametrize("bad, args, why", [
    (dict(), dict(slots=0), b"slots"), (dict(), dict(capacity=7), b"capacity"), (dict(), dict(capacity=100004), b"capacity"),
    (dict(), dict(capacity=(1 << 22) + 8), b"capacity"), (dict(n_samples=479), dict(), b"n_samples"), (dict(min_delay=-1), dict(), b"delays"),
    (dict(min_delay=5, max_delay=4), dict(), b"delays"), (dict(max_delay=(1 << 22) + 1), dict(), b"delays"),
    (dict(max_delay=96001), dict(capacity=120000), b"L_ref"), (dict(n_samples=1 << 22, max_delay=1), dict(capacity=1 << 22), b"L_ref"),
    (dict(), dict(blob=None), b"model"), (dict(), dict(), b"needs a handle")])
def test_every_out_of_range_rule_field_is_refused_before_device_work(bad, args, why):
    from microwakeword_b200 import _lib
    L = _lib.lib()
    g = ctypes.c_void_p(1)
    r = rule(**bad)
    blob = args.get("blob", b"x" * 16)
    rc = L.mww_playback_guard_create(None, blob, 0 if blob is None else len(blob), args.get("slots", 4), 4, args.get("capacity", 160000),
                                     ctypes.byref(r), ctypes.byref(g))
    assert rc == -1 and g.value is None and why in L.mww_last_error(None), (bad, args, L.mww_last_error(None))
    assert L.mww_playback_guard_create(None, blob, 16, 4, 4, 160000, None, ctypes.byref(g)) == -1
    assert L.mww_playback_guard_create(None, blob, 16, 4, 4, 160000, ctypes.byref(r), None) == -1


def test_null_guards_are_refused_without_device_work():
    from microwakeword_b200 import _lib
    L = _lib.lib()
    assert L.mww_playback_guard_destroy(None) == 0
    assert L.mww_playback_guard_info(None, None) == -1
    assert L.mww_playback_write(None, None, None, 0, None, 0, 0, None) == -1
    assert L.mww_playback_read(None, None, None, 0, 0, None, 0, None) == -1
    assert L.mww_playback_reset(None, None, 0, None) == -1
    assert L.mww_playback_get_heads(None, None, None) == -1
    assert L.mww_playback_check_streams(None, None, None, 0, None, None, None, None, None) == -1
    assert L.mww_playback_check_detections_at(None, None, -1, 0, None, None, None, None, None) == -1


def test_python_refusals_before_the_library_is_called(monkeypatch):
    from microwakeword_b200 import _lib
    from microwakeword_b200.playback import PlaybackGuard

    def no_lib():
        raise AssertionError("the library was called")
    monkeypatch.setattr(_lib, "lib", no_lib)
    eng = types.SimpleNamespace(n_streams=8, audio_history_capacity=32000, device=0, _h=None)
    for bad in (dict(slots=0), dict(slots=1.5), dict(rows=0), dict(rows=9), dict(capacity_s=0.0), dict(capacity_s=300.0),
                dict(n_samples=479), dict(min_delay=-1), dict(min_delay=10, max_delay=9), dict(max_delay=(1 << 22) + 1),
                dict(capacity_s=1.0, max_delay=1), dict(window=0), dict(window=33), dict(ignore_steps=-1), dict(cutoff=float("nan")),
                dict(cutoff=True), dict(max_delay=True)):
        kw = dict(slots=4)
        kw.update(bad)
        with pytest.raises(ValueError):
            PlaybackGuard(b"model", eng, **kw)
    with pytest.raises(ValueError):
        PlaybackGuard(b"model", types.SimpleNamespace(n_streams=8, audio_history_capacity=0, device=0, _h=None), slots=4)
    with pytest.raises(ValueError):
        PlaybackGuard(None, eng, slots=4)


def _cuobjdump():
    from microwakeword_b200 import _lib, build
    tool = os.path.join(os.path.dirname(build.NVCC), "cuobjdump")
    if not os.path.exists(tool):
        pytest.skip("cuobjdump is not installed next to nvcc")
    _lib.lib()
    return tool


def test_every_existing_kernel_keeps_its_instructions():
    from microwakeword_b200 import build
    from test_event_positions import _sass_hashes
    before = json.load(open(os.path.join(GOLDEN, "sass_kernels_before_playback_guard.json")))
    libs = [k for k in before if k != "_comment"]
    assert len(libs) == 15 and "libmww_media_guard.so" in libs
    _cuobjdump()
    for lib in libs:
        assert _sass_hashes(os.path.join(os.path.dirname(build.OUT), lib)) == before[lib], lib


def test_companion_library_holds_exactly_its_kernels_without_stack_local_memory_or_spills(monkeypatch):
    from microwakeword_b200 import build
    assert os.path.basename(build.PB_OUT) == "libmww_playback.so" and build.PB_SOURCES == ["mww_playback.cu"]
    res = subprocess.run([_cuobjdump(), "-res-usage", build.PB_OUT], capture_output=True, text=True, check=True).stdout
    found = re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", res)
    names = sorted(re.sub(r".*playback_(\w+?)_kernel.*", r"\1", n) for n, *_ in found)
    assert names == ["decide", "slots", "write"], res
    assert all(int(stack) == int(local) == 0 for _, _, stack, local in found), found
    flags = [f for f in build.FLAGS if f not in ("-shared", "-cudart", "static")]
    rep = subprocess.run([build.NVCC] + flags + ["-cubin", "-Xptxas", "-v", "-o", os.path.join(_BUILD.name, "pb.cubin"),
                                                 os.path.join(CSRC, "mww_playback.cu")], capture_output=True, text=True, check=True).stderr
    spills = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", rep)
    assert len(spills) == 3 and all(int(a) == int(b) == int(c) == 0 for a, b, c in spills), rep
    dyn = subprocess.run(["readelf", "-d", build.OUT], capture_output=True, text=True).stdout
    assert "[libmww_playback.so]" in dyn
    real = os.path.exists
    monkeypatch.setattr(build.os.path, "exists", lambda p: p != build.PB_OUT and real(p))
    assert build._stale()
