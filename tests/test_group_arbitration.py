"""Group arbitration (include/mww.h, "group arbitration"), the parts that need no GPU: the header bodies built with g++ (with
-ffp-contract=off) from microwakeword_b200/csrc/mww_group_arbitration.h by tests/emul_group_arbitration.cc against the NumPy
statement of the rule in tests/group_arbitration_ref.py -- levels on seeded rings, spans that straddle S - C, full-scale
-32768 spans at Ls = 2^20, a large DC offset and all-zero noise, bit for bit; every tie level (level, score, position, row) in
every arrival order, multi-update windows, flush and a checkpoint round trip of windows and levels.  Also the structs, the new
symbols and their argument types, the refusals that need no device, the new library's kernels without stack, local memory or
spills, and every pre-existing kernel's instructions against tests/golden/sass_kernels_before_group_arbitration.json (the
parent's build)."""

import ctypes
import itertools
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
import group_arbitration_ref as ref  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(ROOT, "microwakeword_b200", "csrc")
_BUILD = tempfile.TemporaryDirectory(prefix="mww_group_arbitration_test_")
_emul = []
vp, i32, ll = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong
WINDOW = np.dtype([("deadline", np.int64), ("sample", np.int64), ("step", np.int64), ("stream", np.int32), ("score", np.float32),
                   ("candidates", np.int32), ("open", np.int32)])


def emul():
    if not _emul:
        so = os.path.join(_BUILD.name, "libemul_group_arbitration.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-o", so,
                        os.path.join(HERE, "emul_group_arbitration.cc")], check=True)
        L = ctypes.CDLL(so)
        L.emul_sizes.argtypes = [ctypes.POINTER(i32)] * 3
        L.emul_pending_init.argtypes = [vp, i32]
        L.emul_pending_init.restype = None
        L.emul_levels.argtypes = [vp, i32, ll, vp, vp, i32, i32, i32, vp]
        L.emul_levels.restype = None
        L.emul_energy.argtypes = [ctypes.c_ulonglong, ll, i32]
        L.emul_energy.restype = ctypes.c_double
        L.emul_arbitrated_update.restype = ll
        L.emul_arbitrated_update.argtypes = [i32, ll, vp, vp, vp, i32, vp, vp, vp, vp, vp, vp, vp, ll, ll, i32, i32, vp, i32, vp, vp, vp, vp, vp,
                                             vp, vp]
        _emul.append(L)
    return _emul[0]


def test_struct_sizes_match_the_header():
    p, w, k = i32(), i32(), i32()
    emul().emul_sizes(ctypes.byref(p), ctypes.byref(w), ctypes.byref(k))
    assert (p.value, w.value, k.value) == (32, WINDOW.itemsize, 16) == (32, 40, 16)


# ---- the level -------------------------------------------------------------------------------------------------------------------------
def levels(ring, S, ids, P, Ls, Ln):
    ids, P = np.ascontiguousarray(ids, np.int32), np.ascontiguousarray(P, np.int64)
    out = np.zeros(ids.size, np.float32)
    ring = np.ascontiguousarray(ring, np.int16)
    emul().emul_levels(ring.ctypes.data, ring.shape[1], S, ids.ctypes.data, P.ctypes.data, ids.size, Ls, Ln, out.ctypes.data)
    want = np.array([ref.level(ring, S, int(s), int(p), Ls, Ln) for s, p in zip(ids, P)], np.float32)
    assert np.array_equal(out.view(np.uint32), want.view(np.uint32)), (out, want)
    return out


@pytest.mark.parametrize("seed", range(4))
def test_levels_on_seeded_rings_are_the_rule_bit_for_bit(seed):
    rng = np.random.default_rng(seed)
    C = int(rng.choice([1024, 2000, 4096]))
    ring = (rng.normal(0, rng.uniform(10, 8000), (6, C)) + rng.integers(-3000, 3000, (6, 1))).clip(-32768, 32767).astype(np.int16)
    S = int(rng.integers(C // 2, 5 * C))
    Ls, Ln = int(rng.integers(480, C // 2)), int(rng.integers(480, C // 2))
    P = S - rng.integers(-40, C, 64)                          # spans inside the ring, straddling S - C, past S, before 0
    out = levels(ring, S, rng.integers(0, 6, 64), P, Ls, Ln)
    assert np.isfinite(out).all() and (out > 0).all()


def test_spans_straddling_s_minus_c_read_zeros_outside():
    C, Ls, Ln = 1024, 480, 480
    ring = np.full((1, C), 1000, np.int16)
    S = 5000
    for P in (S - C + Ls, S - C + Ls + Ln - 1, S - C + Ls + Ln, S - C + Ls + Ln + 1, S - C + 100, S - C + 1, S + 200, S + Ls):
        levels(ring, S, [0], [P], Ls, Ln)
    # speech held in full, noise half zeros: a step in the noise span makes it non-stationary
    out = levels(ring, S, [0, 0], [S - C + Ls + Ln, S - C + Ls + Ln // 2], Ls, Ln)
    assert out[0] == np.float32(1.0) and out[1] < 1e-5


def test_full_scale_spans_at_the_largest_length():
    Ls = Ln = 1 << 20
    C = Ls + Ln
    ring = np.full((2, C), -32768, np.int16)
    ring[1, : C // 2] = 0                                           # stream 1: speech full scale -32768 after all-zero noise
    ring[1, C // 2:] = np.where(np.arange(C // 2) % 2, -32768, 32767)
    out = levels(ring, C, [0, 1], [C, C], Ls, Ln)
    assert out[0] == np.float32(1.0)                                # a constant -32768 has no power about its mean
    assert out[1] > 1e9


def test_a_dc_offset_does_not_make_a_device_loud():
    rng = np.random.default_rng(7)
    C, Ls, Ln = 4096, 1000, 1000
    noise = rng.normal(0, 100, C)
    ring = np.stack([noise, noise + 20000]).clip(-32768, 32767).astype(np.int16)
    out = levels(ring, C, [0, 1], [C, C], Ls, Ln)
    assert abs(float(out[0]) - float(out[1])) < 1e-3


def test_all_zero_noise_divides_by_one():
    C, Ls, Ln = 2048, 1000, 1000
    ring = np.zeros((1, C), np.int16)
    ring[0, C - Ls:] = np.where(np.arange(Ls) % 2, 300, -300)
    out = levels(ring, C, [0], [C], Ls, Ln)
    assert out[0] == np.float32(300.0 * 300.0 + 1.0)


def test_energy_arithmetic_edges():
    for q, r, L in ((0, 0, 480), (480 * 2 ** 30, -480 * 2 ** 15, 480), (2 ** 50, -(2 ** 35), 2 ** 20), (12345678901, 987654, 1 << 20),
                    (3, 1, 3), (2 ** 52 + 1, 2 ** 36 - 1, (1 << 20) - 1)):
        got = emul().emul_energy(q, r, L)
        Lf = np.float64(L)
        want = (np.float64(q) - np.float64(r) * np.float64(r) / Lf) / Lf
        assert np.float64(got).view(np.uint64) == want.view(np.uint64), (q, r, L)


# ---- the window rule -------------------------------------------------------------------------------------------------------------------
class Emul:
    """the header bodies over n_slots group slots of one plain detector, with its event buffer"""

    def __init__(self, n_slots, W, capacity, stream_of):
        self.n_slots, self.W, self.capacity = n_slots, W, capacity
        self.stream_of = np.ascontiguousarray(stream_of, np.int32)
        self.pending = np.zeros(n_slots * 32, np.uint8)
        emul().emul_pending_init(self.pending.ctypes.data, n_slots)
        self.windows = np.zeros(n_slots, WINDOW)
        self.levels = np.zeros(n_slots, np.float32)
        self.count = np.zeros(1, np.int64)
        self.out = {k: np.zeros(capacity, t) for k, t in (("sample", np.int64), ("step", np.int64), ("stream", np.int32), ("score", np.float32),
                                                         ("group", np.int32), ("candidates", np.int32), ("level", np.float32))}

    def update(self, cands, seen_after, last_end, step_samples, n, flush=False):
        c = {k: np.ascontiguousarray([x[k] for x in cands], t) for k, t in (("slot", np.int32), ("t", np.int32), ("level", np.float32),
                                                                          ("score", np.float32), ("row", np.int32))}
        o = self.out
        emul().emul_arbitrated_update(self.n_slots, self.W, self.pending.ctypes.data, self.windows.ctypes.data, self.levels.ctypes.data,
                                      len(cands), c["slot"].ctypes.data, c["t"].ctypes.data, c["level"].ctypes.data, c["score"].ctypes.data,
                                      c["row"].ctypes.data, self.stream_of.ctypes.data, seen_after.ctypes.data, last_end, step_samples, n,
                                      int(flush), self.count.ctypes.data, self.capacity, o["sample"].ctypes.data, o["step"].ctypes.data,
                                      o["stream"].ctypes.data, o["score"].ctypes.data, o["group"].ctypes.data, o["candidates"].ctypes.data,
                                      o["level"].ctypes.data)

    def events(self):
        m = min(int(self.count[0]), self.capacity)
        return sorted(zip(*(self.out[k][:m].tolist() for k in ("group", "sample", "stream", "step", "score", "candidates", "level"))))


def key(e):
    return (int(e["group"]), int(e["sample"]), int(e["stream"]), int(e["step"]), float(np.float32(e["score"])), int(e["candidates"]),
            float(np.float32(e["level"])))


def scenario(seed, W, step_samples, n_rows=40, n_slots=7, updates=60, checkpoint_at=None, flush_every=0):
    """one seeded candidate stream through the emulation and the NumPy rule; levels and scores from a few exact values, so that
    every tie level is reached.  checkpoint_at: the windows and levels move to a fresh emulation after that update"""
    rng = np.random.default_rng(seed)
    streams = rng.integers(0, n_rows // 2, n_rows)
    groups = rng.integers(-1, n_slots, n_rows)
    seen = rng.integers(0, 1000, n_rows).astype(np.int64)
    vals = np.float32([0.5, 0.75, 1.0, 4.0])
    em, rule = Emul(n_slots, W, 10 ** 6, streams), ref.ArbRule(W)
    want, last_end = [], int(rng.integers(-10 ** 6, 10 ** 6))
    for u in range(updates):
        n = int(rng.choice([1, 1, 1, 2, 5, 40]))
        last_end += int(rng.integers(1, 3)) * step_samples * n
        if rng.random() < 0.2:
            r = rng.choice(n_rows, 5, replace=False)
            groups[r] = rng.integers(-1, n_slots, 5)
        cands, by_key = [], {}
        for row in range(n_rows):
            for t in range(n):
                if groups[row] < 0 or rng.random() > 0.06:
                    continue
                c = dict(slot=int(groups[row]), t=t, level=vals[rng.integers(0, 4)], score=vals[rng.integers(0, 3)], row=row, id=row,
                         stream=int(streams[row]), sample=last_end - (n - 1 - t) * step_samples, step=int(seen[row]) + t)
                cands.append(c)
                by_key.setdefault(int(groups[row]), []).append(c)
        seen += n
        em.update([cands[i] for i in rng.permutation(len(cands))], seen, last_end, step_samples, n)
        want += rule.update(by_key, last_end - (n - 1) * step_samples, last_end + step_samples)
        if checkpoint_at == u:                                   # the checkpoint: windows and levels into a fresh detector
            moved = Emul(n_slots, W, 10 ** 6, streams)
            moved.windows[:], moved.levels[:] = em.windows, em.levels
            moved.count[:], moved.out = em.count, em.out
            em = moved
        if flush_every and u % flush_every == flush_every - 1:
            em.update([], seen, 0, 1, 0, flush=True)
            want += rule.flush()
    em.update([], seen, 0, 1, 0, flush=True)
    want += rule.flush()
    return em, sorted(key(e) for e in want)


@pytest.mark.parametrize("W,step_samples", [(0, 480), (480, 480), (2000, 480), (3, 1), (7, 1), (2 ** 22, 480)])
def test_emulated_bodies_are_the_rule(W, step_samples):
    total, merged = 0, 0
    for seed in range(6):
        em, want = scenario(100 * W + seed, W, step_samples, flush_every=17 if seed % 2 else 0, checkpoint_at=30 if seed % 3 == 0 else None)
        got = em.events()
        assert got == want, (W, step_samples, seed)
        total += len(want)
        merged += sum(e[5] > 1 for e in want)
    assert total > 50 and (merged > 10 or W == 0)


def test_every_tie_level_in_every_arrival_order():
    """level first, then score, then the earliest step, then the lowest row -- whatever order the offers arrive in"""
    seen = np.full(8, 10, np.int64)
    stream_of = np.array([7, 6, 5, 4, 3, 2, 1, 0], np.int32)
    f = np.float32
    cases = [
        ([dict(t=1, level=f(2), score=f(0.5), row=3), dict(t=0, level=f(1), score=f(1.0), row=0)], (3, 2.0, 0.5, 1)),
        ([dict(t=1, level=f(2), score=f(0.5), row=3), dict(t=1, level=f(2), score=f(0.75), row=4)], (4, 2.0, 0.75, 1)),
        ([dict(t=2, level=f(2), score=f(0.5), row=1), dict(t=1, level=f(2), score=f(0.5), row=6)], (6, 2.0, 0.5, 1)),
        ([dict(t=1, level=f(2), score=f(0.5), row=5), dict(t=1, level=f(2), score=f(0.5), row=2)], (2, 2.0, 0.5, 1)),
        ([dict(t=0, level=f(3), score=f(0.25), row=7), dict(t=2, level=f(3), score=f(0.25), row=0), dict(t=0, level=f(3), score=f(0.25), row=4),
          dict(t=0, level=f(1), score=f(1.0), row=1)], (4, 3.0, 0.25, 0)),
    ]
    for cands, (row, level, score, t) in cases:
        for order in itertools.permutations(range(len(cands))):
            em = Emul(1, 0, 10, stream_of)
            em.update([dict(cands[i], slot=0) for i in order], seen, 1000, 10, 3)
            (e,) = em.events()
            assert (e[2], e[6], e[4], e[1], e[3]) == (stream_of[row], level, score, 1000 - (2 - t) * 10, 10 - 3 + t)


def test_an_exact_tie_across_updates_keeps_the_earlier_candidate():
    stream_of = np.arange(4, dtype=np.int32)
    f = np.float32
    em, rule = Emul(1, 100, 10, stream_of), ref.ArbRule(100)
    seen = np.zeros(4, np.int64)
    steps = [(10, [dict(t=0, level=f(2), score=f(0.5), row=3)]), (20, [dict(t=0, level=f(2), score=f(0.5), row=0)]),
             (30, [dict(t=0, level=f(2), score=f(0.75), row=1)]), (40, [dict(t=0, level=f(4), score=f(0.25), row=2)]),
             (50, [dict(t=0, level=f(4), score=f(0.25), row=0)])]
    want = []
    for last_end, cs in steps:
        seen += 1
        cs = [dict(c, slot=0, id=c["row"], stream=c["row"], sample=last_end, step=int(seen[c["row"]]) - 1) for c in cs]
        em.update(cs, seen, last_end, 10, 1)
        want += rule.update({0: cs}, last_end, last_end + 10)
    em.update([], seen, 0, 1, 0, flush=True)
    want += rule.flush()
    (e,) = em.events()
    assert e == sorted(key(w) for w in want)[0] and (e[2], e[1], e[6], e[5]) == (2, 40, 4.0, 5)


# ---- build, ABI and refusals ----------------------------------------------------------------------------------------------------------
NEW = {"mww_arbitrate_detector_groups": ("mww_detector_t *d, mww_t *src, int speech_samples, int noise_samples", [vp, vp, i32, i32]),
       "mww_drain_detector_arbitrated": ("mww_detector_t *d, mww_event *h_events, int64_t *h_positions, int32_t *h_groups, int32_t *h_candidates, "
                                         "float *h_levels, int max_events, long long *n_events, void *cu_stream",
                                         [vp, vp, vp, vp, vp, vp, i32, ctypes.POINTER(ll), vp]),
       "mww_get_detector_group_levels": ("mww_detector_t *d, float *h_levels", [vp, vp]),
       "mww_set_detector_group_levels": ("mww_detector_t *d, const float *h_levels", [vp, vp])}


def test_new_symbols_are_declared_and_exported_with_their_arguments():
    from microwakeword_b200 import _lib, build
    L = _lib.lib()
    syms = subprocess.run(["nm", "-D", "--defined-only", build.OUT], capture_output=True, text=True, check=True).stdout
    hdr = re.sub(r"\s+", " ", open(os.path.join(ROOT, "include", "mww.h")).read())
    for name, (sig, args) in NEW.items():
        assert name in _lib.EXPORTS and re.search(r"\bT %s\b" % name, syms), name
        assert "int %s(%s);" % (name, sig) in hdr, name
        assert getattr(L, name).argtypes == args, name
    from microwakeword_b200.detection import EVENT_DTYPE, arbitrated_dtype
    assert arbitrated_dtype(EVENT_DTYPE).names[-4:] == ("sample", "group", "candidates", "level")
    assert arbitrated_dtype(EVENT_DTYPE)["level"] == np.float32


def test_null_detectors_are_refused_without_device_work():
    from microwakeword_b200 import _lib
    L = _lib.lib()
    n = ctypes.c_longlong(0)
    assert L.mww_arbitrate_detector_groups(None, None, 12000, 8000) == -1 and b"NULL" in L.mww_last_error(None)
    assert L.mww_drain_detector_arbitrated(None, None, None, None, None, None, 0, ctypes.byref(n), None) == -1
    assert L.mww_get_detector_group_levels(None, None) == -1 and L.mww_set_detector_group_levels(None, None) == -1


def test_python_refusals_before_the_library_is_called():
    from microwakeword_b200.detection import MultiModelDetector, StreamDetector
    det = StreamDetector.__new__(StreamDetector)
    det.n_groups = 0
    for bad in (dict(speech_samples=True), dict(noise_samples=1.5), dict(speech_samples="12000")):
        with pytest.raises(ValueError, match="integer"):
            det.arbitrate(object(), **bad)
    with pytest.raises(ValueError, match="groups"):
        det.arbitrate(object())
    multi = MultiModelDetector.__new__(MultiModelDetector)
    multi.engine, multi.n_groups = object(), 2
    with pytest.raises(ValueError, match="engine it was made with"):
        multi.arbitrate(object())


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
    before = json.load(open(os.path.join(GOLDEN, "sass_kernels_before_group_arbitration.json")))
    libs = [k for k in before if k != "_comment"]
    assert len(libs) == 16 and "libmww_playback.so" in libs and "libmww_detector_groups.so" in libs
    _cuobjdump()
    for lib in libs:
        assert _sass_hashes(os.path.join(os.path.dirname(build.OUT), lib)) == before[lib], lib


def test_companion_library_holds_exactly_its_kernels_without_stack_local_memory_or_spills(monkeypatch):
    from microwakeword_b200 import build
    assert os.path.basename(build.ARB_OUT) == "libmww_group_arbitration.so" and build.ARB_SOURCES == ["mww_group_arbitration.cu"]
    res = subprocess.run([_cuobjdump(), "-res-usage", build.ARB_OUT], capture_output=True, text=True, check=True).stdout
    found = re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", res)
    names = [n for n, *_ in found]
    assert len(names) == 8, res
    assert sum("detector_update_arbitrated_kernel" in n for n in names) == 4
    assert sum("detector_models_update_arbitrated_kernel" in n for n in names) == 2
    assert sum("detector_arbitrated_close_kernel" in n for n in names) == 1
    assert sum("detector_models_arbitrated_close_kernel" in n for n in names) == 1
    assert all(int(stack) == int(local) == 0 for _, _, stack, local in found), found
    flags = [f for f in build.FLAGS if f not in ("-shared", "-cudart", "static")]
    rep = subprocess.run([build.NVCC] + flags + ["-cubin", "-Xptxas", "-v", "-o", os.path.join(_BUILD.name, "arb.cubin"),
                                                 os.path.join(CSRC, "mww_group_arbitration.cu")], capture_output=True, text=True, check=True).stderr
    spills = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", rep)
    assert len(spills) == 8 and all(int(a) == int(b) == int(c) == 0 for a, b, c in spills), rep
    dyn = subprocess.run(["readelf", "-d", build.OUT], capture_output=True, text=True).stdout
    assert "[libmww_group_arbitration.so]" in dyn
    real = os.path.exists
    monkeypatch.setattr(build.os.path, "exists", lambda p: p != build.ARB_OUT and real(p))
    assert build._stale()
