"""The media guard (include/mww.h, "media guard"), the parts that need no GPU: the header bodies built with g++ from
microwakeword_b200/csrc/mww_media_guard.h by tests/emul_media_guard.cc against the NumPy statement of the rule in
tests/media_guard_ref.py -- fingerprints of seeded feature rows, and checks of seeded fingerprints at every edge (the BER bound
and one mismatch more, O == min_overlap and one less, lags at and past max_lag, |dP| at and past the window, households, invalid
slots with and without confirmed ids, ring wrap-around, registered clips shorter and longer than the clip); the structs, the
new symbols and their argument types; the refusals before any device work, in C and in Python; the new library's kernels
without stack, local memory or spills; and every pre-existing kernel's instructions against
tests/golden/sass_kernels_before_media_guard.json (the parent's build)."""

import ctypes
import json
import os
import re
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from conftest import GOLDEN, ROOT

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import media_guard_ref as ref  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(ROOT, "microwakeword_b200", "csrc")
_BUILD = tempfile.TemporaryDirectory(prefix="mww_media_guard_test_")
_emul = []
vp, i32, ll = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong


def emul():
    if not _emul:
        so = os.path.join(_BUILD.name, "libemul_media_guard.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "emul_media_guard.cc")], check=True)
        L = ctypes.CDLL(so)
        L.emul_sizes.argtypes = [ctypes.POINTER(i32), ctypes.POINTER(i32)]
        L.emul_fingerprint.argtypes = [vp, i32, i32, i32, vp]
        L.emul_fingerprint.restype = None
        L.emul_slots_streams.argtypes = [i32, vp, vp, i32, ll, i32, i32, vp]
        L.emul_slots_streams.restype = None
        L.emul_slots_detector.argtypes = [i32, ll, vp, vp, vp, i32, ll, ll, i32, i32, vp, vp, vp, vp, vp]
        L.emul_slots_detector.restype = None
        L.emul_check.argtypes = [i32, i32, vp, vp, vp, vp, vp, vp, i32, vp, vp, vp, vp, vp, i32, vp, vp, i32, i32, i32, i32, ll, vp, vp, vp]
        L.emul_check.restype = None
        _emul.append(L)
    return _emul[0]


def test_struct_sizes_match_the_header():
    from microwakeword_b200 import _lib
    r, d = i32(), i32()
    emul().emul_sizes(ctypes.byref(r), ctypes.byref(d))
    assert (r.value, d.value) == (ctypes.sizeof(_lib.MwwMediaRule), ctypes.sizeof(_lib.MwwMediaGuardDesc)) == (40, 80)


@pytest.mark.parametrize("T", [2, 3, 148, 997])
def test_fingerprints_are_the_rule(T):
    rng = np.random.default_rng(T)
    feat = rng.integers(0, 1 << 16, (3, T, 40)).astype(np.uint16)
    feat[0, :, ::3] = 0                        # extremes and ties: equal differences give bit 0
    feat[1] = rng.integers(0, 3, (T, 40))
    feat[2, :, :20] = 65535
    fp = np.zeros((3, T - 1), np.uint64)
    emul().emul_fingerprint(feat.ctypes.data, 3, T, T - 1, fp.ctypes.data)
    for s in range(3):
        assert np.array_equal(fp[s], ref.fingerprint(feat[s]))
    assert not (fp >> np.uint64(39)).any()


class Guard:
    """the emulated check and the NumPy rule side by side, over the same seeded fingerprints"""

    def __init__(self, W, max_lag, min_overlap, ber_milli, min_matches, ring, window, clips=()):
        self.W, self.args = W, (max_lag, min_overlap, ber_milli, min_matches, window)
        self.ring = ring
        R = max(ring, 1)
        self.count = np.zeros(1, np.int64)
        self.ring_fp, self.ring_stream = np.zeros((R, W), np.uint64), np.zeros(R, np.int32)
        self.ring_hh, self.ring_pos = np.zeros(R, np.int32), np.zeros(R, np.int64)
        self.clips = [np.ascontiguousarray(c, np.uint64) for c in clips]
        self.ref = ref.Rule(max_lag, min_overlap, ber_milli, min_matches, ring, window)
        self.ref.clips = self.clips

    def check(self, fps, sid, valid, hh, pos, confirmed=None):
        n = len(sid)
        fp = np.ascontiguousarray(fps, np.uint64).reshape(n, self.W)
        sid = np.ascontiguousarray(sid, np.int32)
        valid = np.asarray(valid) & (sid >= 0)                 # a slot without a stream is invalid
        rid = np.where(valid, sid, -1).astype(np.int32)
        hh, pos = np.ascontiguousarray(hh, np.int32), np.ascontiguousarray(pos, np.int64)
        conf = None if confirmed is None else np.ascontiguousarray(confirmed, np.int32)
        cfp = np.concatenate(self.clips) if self.clips else np.zeros(1, np.uint64)
        clen = np.array([len(c) for c in self.clips] or [0], np.int32)
        out = [np.zeros(n, np.int32) for _ in range(3)]
        max_lag, mo, ber, mm, window = self.args
        emul().emul_check(n, self.W, fp.ctypes.data, sid.ctypes.data, rid.ctypes.data, hh.ctypes.data, pos.ctypes.data,
                          None if conf is None else conf.ctypes.data, self.ring, self.count.ctypes.data, self.ring_fp.ctypes.data,
                          self.ring_stream.ctypes.data, self.ring_hh.ctypes.data, self.ring_pos.ctypes.data, len(self.clips),
                          cfp.ctypes.data, clen.ctypes.data, max_lag, mo, ber, mm, window, *(o.ctypes.data for o in out))
        want = self.ref.check(list(fp), sid, valid, hh, pos, conf)
        for got, w in zip(out, want):
            assert np.array_equal(got, w), (got, w)
        # the ring holds the NumPy rule's entries, oldest at count mod ring
        kept = self.ref.ring
        assert self.count[0] >= len(kept)
        for k, (f, s, h, p) in enumerate(kept):
            e = (int(self.count[0]) - len(kept) + k) % self.ring
            assert np.array_equal(self.ring_fp[e], f) and (self.ring_stream[e], self.ring_hh[e], self.ring_pos[e]) == (s, h, p)
        return out


def flip(x, k, rng):
    """x with k bits flipped among bits [0, 39) of its words, each bit at most once"""
    y = x.copy()
    cells = rng.choice(len(x) * 39, k, replace=False)
    for c in cells:
        y[c // 39] ^= np.uint64(1) << np.uint64(c % 39)
    return y


def random_fp(n, rng):
    return rng.integers(0, 1 << 39, n, dtype=np.uint64)


def shifted(x, l, rng, n=None):
    """a fingerprint y of n words with y[t + l] = x[t] where both exist, random elsewhere"""
    n = len(x) if n is None else n
    y = random_fp(n, rng)
    for t in range(len(x)):
        if 0 <= t + l < n:
            y[t + l] = x[t]
    return y


def test_ber_bound_is_exact():
    """W = 40 words, lag 0, O = 40: m 1000 == 300 * 39 * 40 mismatches (468) match, 469 do not"""
    rng = np.random.default_rng(1)
    W, mo = 40, 40
    x = random_fp(W, rng)
    for k, flagged in ((468, True), (469, False)):
        g = Guard(W, 0, mo, 300, 1, 0, 10)
        m, media, passed = g.check([x, flip(x, k, rng)], [0, 1], [True, True], [-1, -1], [0, 0])
        assert list(m) == ([1, 1] if flagged else [0, 0]) and list(passed) == ([-1, -1] if flagged else [0, 1])
        assert list(media) == ([2, 2] if flagged else [0, 0])


def test_overlap_and_lag_edges():
    """a copy shifted by l frames: O = W - |l|; it matches at |l| <= max_lag when O >= min_overlap, and never past max_lag"""
    rng = np.random.default_rng(2)
    W, max_lag = 60, 5
    x = random_fp(W, rng)
    for mo, l, want in ((55, 5, 1), (55, -5, 1), (55, 6, 0), (55, -6, 0), (56, 5, 0), (56, 4, 1), (55, 0, 1)):
        g = Guard(W, max_lag, mo, 0, 1, 0, 10)
        m, _, _ = g.check([x, shifted(x, l, rng)], [0, 1], [True, True], [-1, -1], [0, 0])
        assert list(m) == [want, want], (mo, l)


def test_window_and_household_edges():
    rng = np.random.default_rng(3)
    W = 20
    x = random_fp(W, rng)
    g = Guard(W, 0, 20, 0, 1, 0, 1000)
    # |dP| == window counts, window + 1 does not
    assert list(g.check([x, x, x], [0, 1, 2], [True] * 3, [-1] * 3, [5000, 6000, 6001])[0]) == [1, 2, 1]
    # equal groups are one household; group -1 on one stream is one household; -1 on two streams, or a group against -1, are two
    m, _, _ = g.check([x] * 5, [0, 1, 2, 2, 3], [True] * 5, [7, 7, -1, -1, 8], [0] * 5)
    assert list(m) == [3, 3, 3, 3, 4]


def test_invalid_slots_pass_their_confirmed_id():
    rng = np.random.default_rng(4)
    W = 20
    x = random_fp(W, rng)
    for conf in (None, [10, 11, 12, 13]):
        g = Guard(W, 0, 20, 0, 1, 4, 100)
        m, media, passed = g.check([x] * 4, [0, 1, 2, -1], [True, True, False, False], [-1] * 4, [0] * 4, conf)
        assert list(m) == [1, 1, -1, -1] and list(media) == [2, 2, 0, 0]
        assert list(passed) == ([-1, -1, 2, -1] if conf is None else [-1, -1, 12, 13])
        assert g.count[0] == 2


def test_ring_wraps_in_slot_order_and_matches_later_checks():
    rng = np.random.default_rng(5)
    W = 24
    g = Guard(W, 2, 20, 250, 2, 5, 10 ** 6)
    base = random_fp(W, rng)
    for call in range(6):
        n = int(rng.integers(1, 9))
        fps = [flip(shifted(base, int(rng.integers(-2, 3)), rng), int(rng.integers(0, 60)), rng) if rng.random() < 0.6 else random_fp(W, rng)
               for _ in range(n)]
        valid = rng.random(n) < 0.8
        g.check(fps, rng.integers(0, 50, n), valid, rng.integers(-1, 4, n), rng.integers(0, 10 ** 6, n))
    assert g.count[0] > g.ring


@pytest.mark.parametrize("seed", range(8))
def test_seeded_checks_are_the_rule(seed):
    """broadcast-like clusters (shifted copies with flipped bits) among random fingerprints, over several checks, with
    households, windows, invalid slots, a wrapping ring and registered clips shorter and longer than the clip"""
    rng = np.random.default_rng(100 + seed)
    W = int(rng.choice([8, 30, 147]))
    max_lag = int(rng.integers(0, min(8, W - 1) + 1))
    mo = int(rng.integers(1, W - max_lag + 1))
    ad = random_fp(3 * W, rng)
    clips = [ad, ad[W // 2: W // 2 + max(mo, W // 2)], random_fp(W + 5, rng)]
    g = Guard(W, max_lag, mo, int(rng.choice([0, 150, 300, 500])), int(rng.integers(1, 4)), int(rng.choice([0, 3, 16])),
              int(rng.choice([0, 480, 16000])), clips=clips if seed % 2 else ())
    flagged = 0
    for call in range(4):
        n = int(rng.integers(1, 14))
        fps = []
        for _ in range(n):
            r = rng.random()
            if r < 0.5:
                a = int(rng.integers(0, 2 * W))
                fps.append(flip(shifted(ad[a:a + W], int(rng.integers(-max_lag - 1, max_lag + 2)), rng), int(rng.integers(0, W * 8)), rng))
            else:
                fps.append(random_fp(W, rng))
        conf = rng.integers(-1, 50, n) if rng.random() < 0.5 else None
        _, media, _ = g.check(fps, rng.integers(-1, 40, n), rng.random(n) < 0.85, rng.integers(-1, 5, n),
                              call * 8000 + rng.integers(0, 20000, n), conf)
        flagged += int((media != 0).sum())


def test_slots_hear_only_clips_still_in_the_ring():
    ids = np.array([0, 1, 2, 3, -1, 4], np.int32)
    seen, C, N = 10000, 4000, 1000
    ends = np.array([7000, 6999, 10000, 12000, 9000, 9000], np.int64)   # e - N == S - C is heard, one less is not
    rid = np.zeros(6, np.int32)
    emul().emul_slots_streams(6, ids.ctypes.data, ends.ctypes.data, 4, seen, C, N, rid.ctypes.data)
    assert list(rid) == [0, -1, 2, 3, -1, -1]


EVENT = np.dtype([("stream", np.int32), ("reserved", np.int32), ("step", np.int64), ("score", np.float32), ("pad", np.int32)])


def slots_detector(events, count, positions, ev_group, model, post, seen, C, n_samples):
    cap = events.size
    out = [np.zeros(cap, np.int32) for _ in range(3)] + [np.zeros(cap, np.int64) for _ in range(2)]
    emul().emul_slots_detector(cap, count, events.ctypes.data, positions.ctypes.data, None if ev_group is None else ev_group.ctypes.data, model,
                               post, seen, C, n_samples, *(o.ctypes.data for o in out))
    return dict(zip(("sid", "rid", "hh", "end", "pos"), out))


def test_detector_slots_take_the_verifier_rule_with_positions_and_groups():
    """slot i of a timed detector: an unused slot and another model's event give sid = rid = -1; a clip that has partly left
    the ring keeps its stream (it passes) but is not heard; e = min(P + post, S); the household is the event's group, -1 when
    the detector is not grouped"""
    seen, C, N, post = 100000, 40000, 24000, 3200
    ev = np.zeros(8, EVENT)
    ev["stream"] = [10, 11, 12, 13, 14, 15, 16, 17]
    ev["reserved"] = [0, 1, 0, 0, 0, 1, 0, 0]                  # slots 1 and 5 hold model 1's events
    pos = np.array([90000, 90000, seen - 1000, seen - C + N - post, seen - C + N - post - 1, 90000, 85000, 80000], np.int64)
    grp = np.array([3, 4, 5, -1, 6, 7, 8, 9], np.int32)
    count = 7                                                  # slot 7 is unused
    got = slots_detector(ev, count, pos, grp, 0, post, seen, C, N)
    assert list(got["sid"]) == [10, -1, 12, 13, 14, -1, 16, -1]
    assert list(got["rid"]) == [10, -1, 12, 13, -1, -1, 16, -1]      # slot 4: e - N = S - C - 1, left the ring
    assert got["end"][0] == 93200 and got["end"][2] == seen and got["end"][3] == seen - C + N   # slot 2: P + post clamped at S
    assert list(got["hh"][[0, 2, 3, 6]]) == [3, 5, -1, 8] and list(got["pos"][[0, 2, 6]]) == [90000, seen - 1000, 85000]
    any_model = slots_detector(ev, count, pos, None, -1, post, seen, C, N)
    assert list(any_model["sid"]) == [10, 11, 12, 13, 14, 15, 16, -1] and (any_model["hh"][any_model["sid"] >= 0] == -1).all()
    assert list(slots_detector(ev, 100, pos, grp, 1, 0, seen, C, N)["rid"]) == [-1, 11, -1, -1, -1, 15, -1, -1]  # count past capacity


# ---- build, ABI and refusals ----------------------------------------------------------------------------------------------------------
NEW = {"mww_media_guard_create": ("int device, int slots, const mww_media_rule *rule, mww_media_guard_t **out", [i32, i32, None, None]),
       "mww_media_guard_destroy": ("mww_media_guard_t *g", [vp]),
       "mww_media_guard_info": ("const mww_media_guard_t *g, mww_media_guard_desc *out", [vp, None]),
       "mww_media_check_streams": ("mww_media_guard_t *g, mww_t *src, const int32_t *d_ids, const long long *d_ends, const int32_t *d_households, "
                                   "int n, const int32_t *d_confirmed, int32_t *d_matches, int32_t *d_media, int32_t *d_passed, void *cu_stream",
                                   [vp, vp, vp, vp, vp, i32, vp, vp, vp, vp, vp]),
       "mww_media_check_detections_at": ("mww_media_guard_t *g, mww_t *src, mww_detector_t *det, int model, long long post, "
                                         "const int32_t *d_confirmed, int32_t *d_matches, int32_t *d_media, int32_t *d_passed, void *cu_stream",
                                         [vp, vp, vp, i32, ll, vp, vp, vp, vp, vp]),
       "mww_media_register": ("mww_media_guard_t *g, const int16_t *d_audio, int n_samples, int *index, void *cu_stream", [vp, vp, i32, None, vp]),
       "mww_media_clear_registered": ("mww_media_guard_t *g", [vp]),
       "mww_media_clear_ring": ("mww_media_guard_t *g", [vp]),
       "mww_media_get_state": ("mww_media_guard_t *g, void *h_state, long long *n_bytes", [vp, vp, None]),
       "mww_media_set_state": ("mww_media_guard_t *g, const void *h_state, long long n_bytes", [vp, vp, ll])}


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
    r = dict(n_samples=24000, max_lag=15, min_overlap=132, max_ber_milli=300, min_matches=3, ring=8192, max_media=16, max_media_samples=480000,
             window_samples=960000)
    r.update(kw)
    return _lib.MwwMediaRule(*(r[k] for k, _ in _lib.MwwMediaRule._fields_))


@pytest.mark.parametrize("bad", [dict(n_samples=639), dict(n_samples=160001), dict(max_lag=-1), dict(max_lag=65), dict(min_overlap=0),
                                 dict(min_overlap=148), dict(min_overlap=133), dict(max_ber_milli=-1), dict(max_ber_milli=501),
                                 dict(min_matches=0), dict(ring=-1), dict(ring=(1 << 20) + 1), dict(window_samples=-1),
                                 dict(window_samples=(1 << 40) + 1), dict(max_media=-1), dict(max_media=4097),
                                 dict(max_media_samples=-1), dict(max_media_samples=(1 << 24) + 1), dict(max_media_samples=639),
                                 dict(max_media_samples=21440), dict(max_media=4096, max_media_samples=1 << 24)])
def test_every_out_of_range_rule_field_is_refused_before_device_work(bad):
    from microwakeword_b200 import _lib
    L = _lib.lib()
    g = ctypes.c_void_p()
    r = rule(**bad)
    assert L.mww_media_guard_create(0, 4, ctypes.byref(r), ctypes.byref(g)) == -1 and g.value is None, bad
    assert L.mww_media_guard_create(0, 0, ctypes.byref(rule()), ctypes.byref(g)) == -1
    assert L.mww_media_guard_create(0, 4, None, ctypes.byref(g)) == -1


def test_edges_of_the_rule_are_accepted_by_the_checks():
    """the largest legal values pass every field check: what remains is the device (MWW_ECUDA on a host without one)"""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present: create would allocate")
    from microwakeword_b200 import _lib
    L = _lib.lib()
    g = ctypes.c_void_p()
    for r in (rule(), rule(n_samples=640, max_lag=0, min_overlap=1, max_media=0, max_media_samples=0),
              rule(max_lag=64, min_overlap=83, max_ber_milli=500, ring=1 << 20, window_samples=1 << 40, max_media=4096, max_media_samples=5200000)):
        assert L.mww_media_guard_create(0, 4, ctypes.byref(r), ctypes.byref(g)) == -3 and b"no CUDA device" in L.mww_last_error(None)


def test_null_guards_are_refused_without_device_work():
    from microwakeword_b200 import _lib
    L = _lib.lib()
    n = ctypes.c_longlong(0)
    idx = ctypes.c_int(0)
    assert L.mww_media_guard_destroy(None) == 0
    assert L.mww_media_guard_info(None, None) == -1
    assert L.mww_media_check_streams(None, None, None, None, None, 0, None, None, None, None, None) == -1
    assert L.mww_media_check_detections_at(None, None, None, -1, 0, None, None, None, None, None) == -1
    assert L.mww_media_register(None, None, 640, ctypes.byref(idx), None) == -1
    assert L.mww_media_clear_registered(None) == -1 and L.mww_media_clear_ring(None) == -1
    assert L.mww_media_get_state(None, None, ctypes.byref(n)) == -1 and L.mww_media_set_state(None, None, 0) == -1


def test_python_refusals_before_the_library_is_called(monkeypatch):
    from microwakeword_b200 import _lib
    from microwakeword_b200.media import MediaGuard

    def no_lib():
        raise AssertionError("the library was called")
    monkeypatch.setattr(_lib, "lib", no_lib)
    for bad in (dict(slots=0), dict(slots=1.5), dict(n_samples=639), dict(max_lag=65), dict(min_overlap=0), dict(min_overlap=133),
                dict(max_ber=0.51), dict(max_ber=float("nan")), dict(min_matches=0), dict(ring=-1), dict(window_s=-1),
                dict(max_media=4097), dict(max_media_s=0.01), dict(max_lag=True)):
        kw = dict(slots=4)
        kw.update(bad)
        with pytest.raises(ValueError):
            MediaGuard(**kw)


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
    before = json.load(open(os.path.join(GOLDEN, "sass_kernels_before_media_guard.json")))
    libs = [k for k in before if k != "_comment"]
    assert len(libs) == 14 and "libmww_detector_groups.so" in libs
    _cuobjdump()
    for lib in libs:
        assert _sass_hashes(os.path.join(os.path.dirname(build.OUT), lib)) == before[lib], lib


def test_companion_library_holds_exactly_its_kernels_without_stack_local_memory_or_spills(monkeypatch):
    from microwakeword_b200 import build
    assert os.path.basename(build.MG_OUT) == "libmww_media_guard.so" and build.MG_SOURCES == ["mww_media_guard.cu"]
    res = subprocess.run([_cuobjdump(), "-res-usage", build.MG_OUT], capture_output=True, text=True, check=True).stdout
    found = re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", res)
    names = sorted(re.sub(r".*media_(\w+?)_kernel.*", r"\1", n) for n, *_ in found)
    assert names == ["decide", "fingerprint", "match", "slots"], res
    assert all(int(stack) == int(local) == 0 for _, _, stack, local in found), found
    flags = [f for f in build.FLAGS if f not in ("-shared", "-cudart", "static")]
    rep = subprocess.run([build.NVCC] + flags + ["-cubin", "-Xptxas", "-v", "-o", os.path.join(_BUILD.name, "mg.cubin"),
                                                 os.path.join(CSRC, "mww_media_guard.cu")], capture_output=True, text=True, check=True).stderr
    spills = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", rep)
    assert len(spills) == 4 and all(int(a) == int(b) == int(c) == 0 for a, b, c in spills), rep
    dyn = subprocess.run(["readelf", "-d", build.OUT], capture_output=True, text=True).stdout
    assert "[libmww_media_guard.so]" in dyn
    real = os.path.exists
    monkeypatch.setattr(build.os.path, "exists", lambda p: p != build.MG_OUT and real(p))
    assert build._stale()
