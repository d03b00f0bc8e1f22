"""The streaming detector (mww_detector_*, StreamDetector), the parts that need no GPU: the NumPy streaming reference
(tests/detector_ref.py) pinned against the reference's own false-accept counts and the offline oracle; the rule of
microwakeword_b200/csrc/mww_detector.h built for the host (tests/emul_detector.cc) in the thread form and, lane by lane, the
warp form, against that reference for every way of splitting a sequence into calls; the C-ABI's symbols, struct size and
argument checks; the loud failure without a GPU; and the register report of the kernels."""

import ctypes
import itertools
import os
import re
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from detector_ref import EVENT, DetectorRef, same_events, same_state

from oracle import detection_ref as D

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(ROOT, "microwakeword_b200", "csrc")
_BUILD = tempfile.TemporaryDirectory(prefix="mww_detector_test_")
_emul = None


def emul():
    global _emul
    if _emul is None:
        so = os.path.join(_BUILD.name, "libemul_detector.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "emul_detector.cc")], check=True)
        _emul = ctypes.CDLL(so)
        vp, i32, ll = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong
        for fn in (_emul.emul_update_thread, _emul.emul_update_warp):
            fn.restype = ll
            fn.argtypes = [i32, ctypes.c_double, i32, vp, vp, vp, vp, i32, i32, ll, vp, i32]
    return _emul


class Emulated:
    """the header's rule on host state, `form` = "thread" or "warp"; the interface of DetectorRef"""

    def __init__(self, form, n_rows, cutoff, window=5, cooldown_slices=25):
        from microwakeword_b200 import _lib
        self.fn = getattr(emul(), "emul_update_" + form)
        self.n_rows, self.cutoff, self.window, self.cooldown_slices = n_rows, cutoff, window, cooldown_slices
        self.hist = np.zeros((n_rows, window - 1), np.float32)
        self.seen = np.zeros(n_rows, np.int64)
        self.cooldown = np.full(n_rows, cooldown_slices, np.int32)
        self.Event = _lib.MwwEvent

    def update(self, probs, pitch=None):
        probs = np.ascontiguousarray(probs, np.float32).reshape(self.n_rows, -1)
        n = probs.shape[1]
        if pitch is not None:                           # rows further apart than n_steps, the gap filled with a large value
            wide = np.full((self.n_rows, pitch), 9.0, np.float32)
            wide[:, :n] = probs
            probs = wide
        cap = self.n_rows * max(n, 1)
        buf = (self.Event * cap)()
        got = self.fn(self.window, self.cutoff, self.cooldown_slices, self.hist.ctypes.data, self.seen.ctypes.data, self.cooldown.ctypes.data,
                      probs.ctypes.data, self.n_rows, n, probs.shape[1], buf, cap)
        ev = np.zeros(got, EVENT)
        for i in range(got):
            ev[i] = (buf[i].stream, buf[i].step, buf[i].score)
            assert buf[i].reserved == 0 and buf[i].pad == 0
        return ev

    def state(self):
        return dict(hist=self.hist.copy(), seen=self.seen.copy(), cooldown=self.cooldown.copy())


# ---- the reference is the rule the offline path and the reference's harness use ---------------------------------------------
def test_reference_gives_the_pinned_false_accepts_per_hour():
    g = np.load(os.path.join(GOLDEN, "detection_golden.npz"))
    offs = np.concatenate([[0], np.cumsum(g["lengths"])])
    tracks = [g["probs"][offs[i]:offs[i + 1]] for i in range(len(g["lengths"]))]
    window, ignore = int(g["window"]), int(g["ignore"])
    duration_h = 0
    for t in tracks:                                    # test.py:119 on the averaged track the reference passes
        duration_h += max(len(t) - window + 1, 0) * int(g["stride"]) * float(g["step_s"]) / 3600.0
    faph = []
    for cutoff in g["cutoffs"]:
        total = 0
        for t in tracks:
            ref = DetectorRef(1, cutoff, window, ignore)
            total += ref.update(t[None, :]).size
        faph.append(total / duration_h)
    assert np.array_equal(np.asarray(faph), g["faph"])


@pytest.mark.parametrize("window", [1, 5, 32])
@pytest.mark.parametrize("cooldown", [0, 1, 25, 75])
def test_reference_counts_equal_the_offline_oracle(window, cooldown):
    rng = np.random.default_rng(100 * window + cooldown)
    lengths = [0, 1, window - 1, window, window + 1, 40, 333]
    cutoffs = [0.3, 0.6, 0.9]
    for n in lengths:
        track = rng.random(n).astype(np.float32)
        want = D.false_accept_counts(D.moving_average(track, window), cutoffs, cooldown)
        for c, w in zip(cutoffs, want):
            ref = DetectorRef(1, c, window, cooldown)
            ev = ref.update(track[None, :])
            assert ev.size == w, (n, c)
            # the event's score is the offline moving average at step - (window - 1)
            avg = D.moving_average(track, window)
            assert np.array_equal(ev["score"], avg[ev["step"] - (window - 1)])


# ---- the header's two forms against the reference, for every split into calls ---------------------------------------------
def splits(total, sizes, limit, rng):
    """call-size sequences summing to `total`: every one-size pattern, and seeded mixtures"""
    out = [[total]]
    for s in sizes:
        if 0 < s <= total:
            out.append([s] * (total // s) + ([total % s] if total % s else []))
    for _ in range(limit):
        seq, left = [], total
        while left:
            s = min(int(rng.choice(sizes)), left)
            seq.append(s)
            left -= s
        out.append(seq)
    return out


def run_split(det, probs, seq, pitch=None):
    evs, at = [], 0
    for n in seq:
        evs.append(det.update(probs[:, at:at + n], pitch=pitch))
        at += n
    assert at == probs.shape[1]
    return np.concatenate(evs) if evs else np.zeros(0, EVENT)


CASES = [(1, 0), (1, 3), (2, 1), (5, 25), (5, 0), (7, 2), (31, 4), (32, 25)]


@pytest.mark.parametrize("window,cooldown", CASES)
def test_both_forms_equal_the_reference_for_every_split(window, cooldown):
    rng = np.random.default_rng(7 * window + cooldown)
    R, total, cutoff = 6, 137, 0.5                      # sums of 0.5 are exact, so row 3 averages exactly the cutoff
    probs = rng.random((R, total)).astype(np.float32)
    probs[1] = 0.99                                     # fires as often as the cooldown allows
    probs[2, 40:44] = np.nan                            # NaN never fires, and is gone once it leaves the history
    probs[3] = np.float32(cutoff)                       # an average equal to the cutoff: no event
    want_ref = DetectorRef(R, cutoff, window, cooldown)
    want = want_ref.update(probs)
    assert want.size > 0 and not (want["stream"] == 3).any()
    sizes = [0, 1, 2, 3, 7, 100]
    for seq in splits(total, sizes, 12, rng):
        for form in ("thread", "warp"):
            det = Emulated(form, R, cutoff, window, cooldown)
            got = run_split(det, probs, seq)
            assert same_events(got, want), (form, seq)
            assert same_state(det.state(), want_ref.state()), (form, seq)


def test_average_equal_to_the_cutoff_does_not_fire_and_one_ulp_above_does():
    window = 4
    p = np.full((1, 12), 0.75, np.float32)
    for form in ("thread", "warp"):
        assert Emulated(form, 1, 0.75, window, 0).update(p).size == 0
        below = float(np.nextafter(np.float32(0.75), np.float32(0)))
        ev = Emulated(form, 1, below, window, 0).update(p)
        assert ev["step"].tolist() == list(range(window - 1, 12)) and (ev["score"] == np.float32(0.75)).all()


def test_tracks_shorter_than_the_window_yield_nothing_until_it_fills():
    for form in ("thread", "warp"):
        det = Emulated(form, 2, 0.1, 5, 0)
        assert det.update(np.ones((2, 4), np.float32)).size == 0 and det.seen.tolist() == [4, 4]
        assert det.cooldown.tolist() == [0, 0]
        ev = det.update(np.ones((2, 1), np.float32))
        assert ev["step"].tolist() == [4, 4]
    # the cooldown does not tick while a row warms up: with 3 slices the first event is at step window - 1 + 2
    for form in ("thread", "warp"):
        ev = Emulated(form, 1, 0.1, 5, 3).update(np.ones((1, 20), np.float32))
        assert ev["step"].tolist() == [6, 9, 12, 15, 18]


def test_pitch_beyond_the_steps_is_not_read():
    rng = np.random.default_rng(3)
    probs = rng.random((4, 50)).astype(np.float32)
    want = DetectorRef(4, 0.5, 5, 2).update(probs)
    for form in ("thread", "warp"):
        got = run_split(Emulated(form, 4, 0.5, 5, 2), probs, [3, 40, 7], pitch=64)
        assert same_events(got, want)


def test_nan_stops_mattering_once_it_leaves_the_history():
    window = 5
    p = np.full((1, 30), 0.9, np.float32)
    p[0, 10] = np.nan
    for form in ("thread", "warp"):
        ev = Emulated(form, 1, 0.5, window, 0).update(p)
        assert ev["step"].tolist() == [s for s in range(window - 1, 30) if not 10 <= s < 10 + window]


def test_chain_over_candidates_equals_the_step_by_step_chain():
    """detector_chain_pass through the warp form on masks of every density, long cooldowns included"""
    rng = np.random.default_rng(11)
    for density, cooldown in itertools.product((0.02, 0.3, 0.9), (0, 1, 5, 31, 32, 33, 200)):
        probs = (rng.random((3, 300)) < density).astype(np.float32)
        want = DetectorRef(3, 0.5, 1, cooldown).update(probs)
        got = run_split(Emulated("warp", 3, 0.5, 1, cooldown), probs, [100, 64, 1, 35, 100])
        assert same_events(got, want), (density, cooldown)


# ---- C-ABI ----------------------------------------------------------------------------------------------------------------
def test_event_struct_is_24_bytes_everywhere():
    from microwakeword_b200 import _lib, detection
    assert ctypes.sizeof(_lib.MwwEvent) == emul().emul_sizeof_event() == detection.EVENT_DTYPE.itemsize == 24
    assert [n for n, _ in _lib.MwwEvent._fields_] == list(detection.EVENT_DTYPE.names)
    assert [detection.EVENT_DTYPE.fields[n][1] for n in detection.EVENT_DTYPE.names] == [getattr(_lib.MwwEvent, n).offset for n in detection.EVENT_DTYPE.names]


def test_detector_symbols_are_exported():
    from microwakeword_b200 import _lib
    L = _lib.lib()
    names = [n for n in _lib.EXPORTS if n.startswith("mww_detector_")]
    assert len(names) == 9
    for n in names:
        assert hasattr(L, n)
    hdr = open(os.path.join(ROOT, "include", "mww.h")).read()
    assert "kDetectorWarpMinSteps = %d" % emul().emul_warp_min_steps() in open(os.path.join(CSRC, "mww_detector.h")).read()
    assert "typedef struct mww_event { int32_t stream, reserved; int64_t step; float score; int32_t pad; } mww_event;" in hdr


def _create(**kw):
    from microwakeword_b200 import _lib
    L = _lib.lib()
    a = dict(device=0, n_rows=8, window=5, cutoff=0.5, cooldown_slices=25, capacity=16)
    a.update(kw)
    d = ctypes.c_void_p()
    rc = L.mww_detector_create(a["device"], a["n_rows"], a["window"], a["cutoff"], a["cooldown_slices"], a["capacity"], None, ctypes.byref(d))
    return rc, (L.mww_last_error(None) or b"").decode(), d


def test_bad_arguments_are_refused_before_any_device_work():
    for bad, word in ((dict(window=0), "window"), (dict(window=33), "window"), (dict(cooldown_slices=-1), "cooldown"),
                      (dict(cutoff=float("nan")), "cutoff"), (dict(cutoff=float("inf")), "cutoff"), (dict(capacity=0), "capacity"),
                      (dict(n_rows=0), "n_rows")):
        rc, msg, d = _create(**bad)
        assert rc == -1 and word in msg and not d.value, bad
    from microwakeword_b200 import _lib
    L = _lib.lib()
    n = ctypes.c_longlong(0)
    assert L.mww_detector_update(None, None, 1, 1, None) == -1
    assert L.mww_detector_drain(None, None, 0, ctypes.byref(n), None) == -1
    assert L.mww_detector_reset(None, None, 0, None) == -1 and L.mww_detector_reset_device(None, None, 0, None) == -1
    assert L.mww_detector_get_state(None, None, None, None) == -1 and L.mww_detector_set_state(None, None, None, None) == -1
    assert L.mww_detector_buffers(None, None, None, None, None) == -1
    assert L.mww_detector_destroy(None) == 0


def test_no_cpu_fallback_without_a_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present; the loud-failure path is exercised on GPU-less hosts")
    rc, msg, d = _create()
    assert rc == -3 and "no CUDA device" in msg and not d.value
    from microwakeword_b200 import _lib
    from microwakeword_b200.detection import StreamDetector
    with pytest.raises(_lib.MwwError) as e:
        StreamDetector(8, cutoff=0.5)
    assert e.value.code == -3 and "no CUDA device" in str(e.value)
    with pytest.raises(ValueError):
        StreamDetector(8, cutoff=0.5, stream_ids=[1, 2, 3])
    tool = os.path.join(ROOT, "tools", "detector_time.py")
    res = subprocess.run([sys.executable, tool, "--rows", "64"], capture_output=True, text=True)
    assert res.returncode != 0 and "CUDA" in res.stderr


# ---- the kernels keep their state in registers --------------------------------------------------------------------------------
def test_detector_kernels_do_not_spill():
    from microwakeword_b200 import build
    if not os.path.exists(build.NVCC):
        pytest.skip("nvcc is not installed")
    flags = [f for f in build.FLAGS if f not in ("-shared", "-cudart", "static")]
    res = subprocess.run([build.NVCC] + flags + ["-cubin", "-Xptxas", "-v", "-o", os.path.join(_BUILD.name, "detector.cubin"),
                                                  os.path.join(CSRC, "mww_detector.cu")], capture_output=True, text=True, check=True)
    reports = re.findall(r"Function properties for (\S+)\s+(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", res.stderr)
    names = sorted(name for name, *_ in reports)
    assert len(names) == 3 and sum("detector_update_kernel" in n for n in names) == 2 and sum("detector_reset_kernel" in n for n in names) == 1, res.stderr
    assert all(int(stack) == int(st) == int(ld) == 0 for _, stack, st, ld in reports), reports


def test_main_library_links_the_detector_library():
    from microwakeword_b200 import build
    assert os.path.basename(build.DET_OUT) == "libmww_detector.so" and build.DET_SOURCES == ["mww_detector.cu"]
    from microwakeword_b200 import _lib
    _lib.lib()
    assert os.path.exists(build.DET_OUT)
    import shutil
    if shutil.which("readelf"):
        dyn = subprocess.run(["readelf", "-d", build.OUT], capture_output=True, text=True, check=True)
        assert "libmww_detector.so" in dyn.stdout and "$ORIGIN" in dyn.stdout
