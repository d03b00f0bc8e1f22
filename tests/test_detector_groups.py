"""Grouped detection (include/mww.h, "grouped detection"), the parts that need no GPU: the rule's bodies (key, offer, close) built
with g++ from microwakeword_b200/csrc/mww_detector_groups.h by tests/emul_detector_groups.cc and checked against the NumPy
statement of the rule in tests/detector_groups_ref.py, on seeded candidate streams that hit exact window boundaries (a
candidate at D - 1 against one at D, a_u = D), every tie level, W = 0, multi-step updates, groups changed while a window is open,
flush and capacity overflow; the new library's kernels without stack, local memory or spills; every pre-existing kernel's
instructions against tests/golden/sass_kernels_before_detector_groups.json (the parent's build); the new symbols and their
argument types; and the refusals that need no device."""

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
from detector_groups_ref import GroupRule  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(ROOT, "microwakeword_b200", "csrc")
_BUILD = tempfile.TemporaryDirectory(prefix="mww_detector_groups_test_")
_emul = []
vp, i32, ll = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong
WINDOW = np.dtype([("deadline", np.int64), ("sample", np.int64), ("step", np.int64), ("stream", np.int32), ("score", np.float32),
                   ("candidates", np.int32), ("open", np.int32)])


def emul():
    if not _emul:
        so = os.path.join(_BUILD.name, "libemul_detector_groups.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "emul_detector_groups.cc")], check=True)
        L = ctypes.CDLL(so)
        L.emul_sizes.argtypes = [ctypes.POINTER(i32), ctypes.POINTER(i32)]
        L.emul_pending_init.argtypes = [vp, i32]
        L.emul_pending_init.restype = None
        L.emul_group_update.restype = ll
        L.emul_group_update.argtypes = [i32, ll, vp, vp, i32, vp, vp, vp, vp, vp, vp, ll, ll, i32, i32, vp, i32, vp, vp, vp, vp, vp, vp]
        _emul.append(L)
    return _emul[0]


def test_struct_sizes_match_the_header():
    p, w = i32(), i32()
    emul().emul_sizes(ctypes.byref(p), ctypes.byref(w))
    assert (p.value, w.value) == (32, WINDOW.itemsize) == (32, 40)


class Emul:
    """the header bodies over n_slots group slots of one plain detector, with its event buffer"""

    def __init__(self, n_slots, W, capacity):
        self.n_slots, self.W, self.capacity = n_slots, W, capacity
        self.pending = np.zeros(n_slots * 32, np.uint8)
        emul().emul_pending_init(self.pending.ctypes.data, n_slots)
        self.windows = np.zeros(n_slots, WINDOW)
        self.count = np.zeros(1, np.int64)
        self.out = {k: np.zeros(capacity, t) for k, t in (("sample", np.int64), ("step", np.int64), ("stream", np.int32), ("score", np.float32),
                                                         ("group", np.int32), ("candidates", np.int32))}

    def update(self, cands, seen_after, last_end, step_samples, n, flush=False):
        c = {k: np.ascontiguousarray([x[k] for x in cands], t) for k, t in (("slot", np.int32), ("t", np.int32), ("score", np.float32),
                                                                          ("stream", np.int32), ("row", np.int32))}
        o = self.out
        emul().emul_group_update(self.n_slots, self.W, self.pending.ctypes.data, self.windows.ctypes.data, len(cands), c["slot"].ctypes.data,
                                 c["t"].ctypes.data, c["score"].ctypes.data, c["stream"].ctypes.data, c["row"].ctypes.data,
                                 seen_after.ctypes.data, last_end, step_samples, n, int(flush), self.count.ctypes.data, self.capacity,
                                 o["sample"].ctypes.data, o["step"].ctypes.data, o["stream"].ctypes.data, o["score"].ctypes.data,
                                 o["group"].ctypes.data, o["candidates"].ctypes.data)

    def events(self):
        m = min(int(self.count[0]), self.capacity)
        return sorted(zip(*(self.out[k][:m].tolist() for k in ("group", "sample", "stream", "step", "score", "candidates"))))


def key(e):
    return (int(e["group"]), int(e["sample"]), int(e["stream"]), int(e["step"]), float(np.float32(e["score"])), int(e["candidates"]))


def scenario(seed, W, step_samples, n_rows=40, n_slots=7, updates=60, capacity=10 ** 6, change_groups=True, flush_every=0):
    """one seeded candidate stream through the emulation and the NumPy rule; -> (emulated, reference) events and the count"""
    rng = np.random.default_rng(seed)
    streams = rng.integers(0, n_rows // 2, n_rows)             # a stream map that repeats ids: the row tie level is reached
    groups = rng.integers(-1, n_slots, n_rows)
    seen = rng.integers(0, 1000, n_rows).astype(np.int64)
    scores = np.float32([0.5, 0.75, 0.875, 1.0])               # a few exact values: score ties are common
    em, ref = Emul(n_slots, W, capacity), GroupRule(W)
    want, last_end = [], int(rng.integers(-10 ** 6, 10 ** 6))
    for u in range(updates):
        n = int(rng.choice([1, 1, 1, 2, 5, 40]))                 # live calls and multi-step ones
        last_end += int(rng.integers(1, 3)) * step_samples * n  # gaps: a_u can be past E_{u-1}
        if change_groups and rng.random() < 0.2:                  # groups change while windows are open
            r = rng.choice(n_rows, 5, replace=False)
            groups[r] = rng.integers(-1, n_slots, 5)
        cands, by_key = [], {}
        for row in range(n_rows):
            for t in range(n):
                if groups[row] < 0 or rng.random() > 0.06:
                    continue
                c = dict(slot=int(groups[row]), t=t, score=scores[rng.integers(0, 4)], stream=int(streams[row]), row=row,
                         sample=last_end - (n - 1 - t) * step_samples, step=int(seen[row]) + t)
                cands.append(c)
                by_key.setdefault(int(groups[row]), []).append(c)
        order = rng.permutation(len(cands))                     # offers arrive in any order
        seen += n
        em.update([cands[i] for i in order], seen, last_end, step_samples, n)
        want += ref.update(by_key, last_end - (n - 1) * step_samples, last_end + step_samples)
        if flush_every and u % flush_every == flush_every - 1:
            em.update([], seen, 0, 1, 0, flush=True)
            want += ref.flush()
    em.update([], seen, 0, 1, 0, flush=True)
    want += ref.flush()
    return em, sorted(key(e) for e in want)


@pytest.mark.parametrize("W,step_samples", [(0, 480), (480, 480), (1440, 480), (2000, 480), (3, 1), (1, 1), (7, 1), (2 ** 22, 480)])
def test_emulated_bodies_are_the_rule(W, step_samples):
    total, merged = 0, 0
    for seed in range(6):
        em, want = scenario(100 * W + seed, W, step_samples, flush_every=17 if seed % 2 else 0)
        got = em.events()
        assert got == want, (W, step_samples, seed)
        total += len(want)
        merged += sum(e[5] > 1 for e in want)
    assert total > 50 and (merged > 10 or W == 0 or W == 1)


def test_window_boundaries_are_exact():
    """step_samples 1: a candidate at D - 1 joins the window, one at D opens the next, and an update whose first step ends at D
    closes the window before its own candidates (a_u = D); E_u = D closes it after them"""
    em, ref = Emul(1, 10, 100), GroupRule(10)
    seen = np.zeros(4, np.int64)

    def up(last_end, n, cands):
        seen[:] += n
        cs = [dict(slot=0, t=t, score=np.float32(s), stream=r, row=r, sample=last_end - (n - 1 - t), step=int(seen[r]) - n + t)
              for t, s, r in cands]
        em.update(cs, seen, last_end, 1, n)
        return ref.update({0: cs} if cs else {}, last_end - (n - 1), last_end + 1)

    want = up(100, 1, [(0, 0.5, 0)])                 # opens: D = 110
    want += up(109, 1, [(0, 0.6, 1)])                # at D - 1: merged (E = 110 closes it)
    want += up(112, 3, [(0, 0.7, 2), (2, 0.9, 3)])   # a_u = 110 = D of nothing open; opens D = 120
    want += up(121, 2, [(1, 0.4, 0)])                # a_u = 120 = D: the window closes first, the candidate opens a new one
    want += ref.flush()
    em.update([], seen, 0, 1, 0, flush=True)
    assert em.events() == sorted(key(e) for e in want)
    got = em.events()
    assert [(g[1], g[5]) for g in got] == [(109, 2), (112, 2), (121, 1)]


def test_every_tie_level_is_decided_by_the_key():
    """equal scores: the earliest step wins; equal score and step: the lowest stream; then the lowest row -- whatever the order"""
    rng = np.random.default_rng(5)
    seen = np.zeros(8, np.int64)
    base = [dict(slot=0, t=2, score=np.float32(0.9), stream=5, row=0), dict(slot=0, t=1, score=np.float32(0.9), stream=6, row=1),
            dict(slot=0, t=1, score=np.float32(0.9), stream=4, row=2), dict(slot=0, t=1, score=np.float32(0.9), stream=4, row=3),
            dict(slot=0, t=0, score=np.float32(0.8), stream=0, row=4), dict(slot=0, t=1, score=np.float32(-0.0), stream=1, row=5)]
    for _ in range(20):
        em = Emul(1, 0, 10)
        em.update([base[i] for i in rng.permutation(len(base))], seen + 3, 1000, 10, 3)
        (e,) = em.events()
        assert (e[2], e[1], e[5]) == (4, 990, 6) and e[3] == 1          # stream 4, step t = 1, row 2 (its step is seen - 3 + 1)


def test_capacity_overflow_is_counted_not_stored():
    em, want = scenario(7, 480, 480, capacity=5)
    assert int(em.count[0]) == len(want) > 5
    assert len(em.events()) == 5 and set(em.events()) <= set(want)


# ---- build, ABI and refusals ----------------------------------------------------------------------------------------------------------
NEW = {"mww_group_detector_events": ("mww_detector_t *d, int n_groups, long long window_samples", [vp, i32, ll]),
       "mww_set_detector_groups": ("mww_detector_t *d, const int32_t *h_rows, const int32_t *h_groups, int n, void *cu_stream", [vp, vp, vp, i32, vp]),
       "mww_get_detector_groups": ("mww_detector_t *d, int32_t *h_groups", [vp, vp]),
       "mww_set_multi_detector_groups": ("mww_detector_t *d, const int32_t *h_stream_ids, const int32_t *h_groups, int n, void *cu_stream",
                                         [vp, vp, vp, i32, vp]),
       "mww_get_multi_detector_groups": ("mww_detector_t *d, int32_t *h_groups", [vp, vp]),
       "mww_flush_detector_groups": ("mww_detector_t *d, void *cu_stream", [vp, vp]),
       "mww_drain_detector_groups": ("mww_detector_t *d, mww_event *h_events, int64_t *h_positions, int32_t *h_groups, int32_t *h_candidates, "
                                     "int max_events, long long *n_events, void *cu_stream", [vp, vp, vp, vp, vp, i32, ctypes.POINTER(ll), vp]),
       "mww_get_detector_group_windows": ("mww_detector_t *d, mww_group_window *h_windows", [vp, vp]),
       "mww_set_detector_group_windows": ("mww_detector_t *d, const mww_group_window *h_windows", [vp, vp])}


def test_new_symbols_are_declared_and_exported_with_their_arguments():
    from microwakeword_b200 import _lib, build
    L = _lib.lib()
    syms = subprocess.run(["nm", "-D", "--defined-only", build.OUT], capture_output=True, text=True, check=True).stdout
    hdr = re.sub(r"\s+", " ", open(os.path.join(ROOT, "include", "mww.h")).read())
    for name, (sig, args) in NEW.items():
        assert name in _lib.EXPORTS and re.search(r"\bT %s\b" % name, syms), name
        assert "int %s(%s);" % (name, sig) in hdr, name
        assert getattr(L, name).argtypes == args, name
    from microwakeword_b200.detection import GROUP_WINDOW_DTYPE
    assert GROUP_WINDOW_DTYPE == WINDOW


def test_null_detectors_are_refused_without_device_work():
    from microwakeword_b200 import _lib
    L = _lib.lib()
    n = ctypes.c_longlong(0)
    assert L.mww_group_detector_events(None, 1, 0) == -1 and b"NULL" in L.mww_last_error(None)
    assert L.mww_set_detector_groups(None, None, None, 0, None) == -1
    assert L.mww_set_multi_detector_groups(None, None, None, 0, None) == -1
    assert L.mww_get_detector_groups(None, None) == -1 and L.mww_get_multi_detector_groups(None, None) == -1
    assert L.mww_flush_detector_groups(None, None) == -1
    assert L.mww_drain_detector_groups(None, None, None, None, None, 0, ctypes.byref(n), None) == -1
    assert L.mww_get_detector_group_windows(None, None) == -1 and L.mww_set_detector_group_windows(None, None) == -1


def test_python_refusals_before_the_library_is_called():
    from microwakeword_b200.detection import MultiModelDetector, StreamDetector, _group_list
    with pytest.raises(ValueError, match="timed"):
        StreamDetector(4, 0.5, groups=2)
    with pytest.raises(ValueError, match="timed"):
        MultiModelDetector(None, [0.5], groups=2)
    for bad in (dict(groups=1.5), dict(groups=True), dict(groups=2, group_window=0.5)):
        with pytest.raises(ValueError, match="integer"):
            StreamDetector(4, 0.5, timed=True, **bad)
    for ids, g in (([[0, 1]], 0), ([0, 1], [0]), ([0, 1], [0.5, 1]), ([0], [2 ** 40])):
        with pytest.raises(ValueError):
            _group_list(ids, g, "rows")


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
    before = json.load(open(os.path.join(GOLDEN, "sass_kernels_before_detector_groups.json")))
    libs = [k for k in before if k != "_comment"]
    assert len(libs) == 13 and "libmww_event_positions.so" in libs
    for lib in libs:
        assert _sass_hashes(os.path.join(os.path.dirname(build.OUT), lib)) == before[lib], lib


def test_companion_library_holds_exactly_its_kernels_without_stack_local_memory_or_spills(monkeypatch):
    from microwakeword_b200 import build
    assert os.path.basename(build.GRP_OUT) == "libmww_detector_groups.so" and build.GRP_SOURCES == ["mww_detector_groups.cu"]
    res = subprocess.run([_cuobjdump(), "-res-usage", build.GRP_OUT], capture_output=True, text=True, check=True).stdout
    found = re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", res)
    names = [n for n, *_ in found]
    assert len(names) == 8, res
    assert sum("detector_update_grouped_kernel" in n for n in names) == 4
    assert sum("detector_models_update_grouped_kernel" in n for n in names) == 2
    assert sum("detector_groups_close_kernel" in n for n in names) == 1 and sum("detector_models_groups_close_kernel" in n for n in names) == 1
    assert all(int(stack) == int(local) == 0 for _, _, stack, local in found), found
    flags = [f for f in build.FLAGS if f not in ("-shared", "-cudart", "static")]
    rep = subprocess.run([build.NVCC] + flags + ["-cubin", "-Xptxas", "-v", "-o", os.path.join(_BUILD.name, "grp.cubin"),
                                                 os.path.join(CSRC, "mww_detector_groups.cu")], capture_output=True, text=True, check=True).stderr
    spills = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", rep)
    assert len(spills) == 8 and all(int(a) == int(b) == int(c) == 0 for a, b, c in spills), rep
    dyn = subprocess.run(["readelf", "-d", build.OUT], capture_output=True, text=True).stdout
    assert "[libmww_detector_groups.so]" in dyn
    real = os.path.exists
    monkeypatch.setattr(build.os.path, "exists", lambda p: p != build.GRP_OUT and real(p))
    assert build._stale()
