"""Second-stage verification (mww_verifier_* / mww_verify_*; microwakeword_b200.verify.Verifier), the parts that need no GPU:
the two kernels' per-element bodies (microwakeword_b200/csrc/mww_verify.h, built with g++ in a temporary directory by
tests/emul_verify.cc) against a NumPy model of the rule in include/mww.h -- the slot rule over event counts of 0, below and
above the capacity, model filters on mixed model tags and stream ids out of range, and the confirm rule on NaN scores and on
cutoffs one double step either side of a float32 score -- the C and Python refusals that fire before any device work, the
refusal of create without a GPU, the symbols and structs, the companion library's link, kernels and registers, and the
timing tool's loud failure without a GPU."""

import ctypes
import os
import re
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from conftest import GOLDEN, ROOT

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(ROOT, "microwakeword_b200", "csrc")
_BUILD = tempfile.TemporaryDirectory(prefix="mww_verify_test_")
_emul = None

EVENT = np.dtype([("stream", np.int32), ("reserved", np.int32), ("step", np.int64), ("score", np.float32), ("pad", np.int32)])


def emul():
    global _emul
    if _emul is None:
        so = os.path.join(_BUILD.name, "libemul_verify.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "emul_verify.cc")], check=True)
        _emul = ctypes.CDLL(so)
        vp, i32 = ctypes.c_void_p, ctypes.c_int
        _emul.emul_verify_slots.restype = None
        _emul.emul_verify_slots.argtypes = [ctypes.c_longlong, vp, i32, i32, vp]
        _emul.emul_verify_confirm.restype = None
        _emul.emul_verify_confirm.argtypes = [vp, i32, i32, vp, ctypes.c_double, vp, vp]
    return _emul


# ---- the rule in NumPy ---------------------------------------------------------------------------------------------------------------
def slots_ref(count, events, capacity, model):
    ids = np.full(capacity, -1, np.int32)
    for i in range(min(count, capacity)):
        if model < 0 or events["reserved"][i] == model:
            ids[i] = events["stream"][i]
    return ids


def confirm_ref(ids, n_streams, scores, cutoff):
    listed = (ids >= 0) & (ids < n_streams)
    out = np.where(listed, scores, np.float32(np.nan)).astype(np.float32)
    ok = listed & (scores.astype(np.float64) > cutoff)          # NaN > x is False
    return out, np.where(ok, ids, -1).astype(np.int32)


def run_slots(count, events, capacity, model):
    ids = np.empty(capacity, np.int32)
    emul().emul_verify_slots(count, events.ctypes.data, capacity, model, ids.ctypes.data)
    return ids


def run_confirm(ids, n_streams, scores, cutoff):
    ids = np.ascontiguousarray(ids, np.int32)
    scores = np.ascontiguousarray(scores, np.float32)
    out_s, out_c = np.empty(ids.size, np.float32), np.empty(ids.size, np.int32)
    emul().emul_verify_confirm(ids.ctypes.data, ids.size, n_streams, scores.ctypes.data, cutoff, out_s.ctypes.data, out_c.ctypes.data)
    return out_s, out_c


def _events(rng, capacity, n_models, n_streams):
    ev = np.zeros(capacity, EVENT)
    ev["stream"] = rng.integers(-3, n_streams + 3, capacity)        # negative and out-of-range ids pass through the slot rule
    ev["reserved"] = rng.integers(0, n_models, capacity)
    ev["step"] = rng.integers(0, 10 ** 6, capacity)
    ev["score"] = rng.random(capacity, dtype=np.float32)
    return ev


@pytest.mark.parametrize("count", [0, 1, 37, 63, 64, 65, 1000])
@pytest.mark.parametrize("model", [-1, 0, 2])
def test_slot_rule(count, model):
    rng = np.random.default_rng(count * 7 + model + 11)
    capacity = 64
    ev = _events(rng, capacity, 3, 100)
    got = run_slots(count, ev, capacity, model)
    want = slots_ref(count, ev, capacity, model)
    assert np.array_equal(got, want)
    used = min(count, capacity)
    assert (got[used:] == -1).all()                                  # slots past the count
    if model < 0:
        assert np.array_equal(got[:used], ev["stream"][:used])
    else:
        assert ((got[:used] == -1) | (ev["reserved"][:used] == model)).all()


def test_slot_rule_model_filters_partition_the_used_slots():
    rng = np.random.default_rng(5)
    ev = _events(rng, 200, 4, 50)
    ev["stream"] = np.arange(200)
    for count in (0, 150, 200, 10 ** 9):
        every = run_slots(count, ev, 200, -1)
        parts = [run_slots(count, ev, 200, k) for k in range(4)]
        merged = np.max(np.stack(parts), 0)                              # each used slot belongs to exactly one model
        assert np.array_equal(merged, every)
        assert (np.sum(np.stack(parts) >= 0, 0) == (every >= 0)).all()
        assert (run_slots(count, ev, 200, 4) == -1).all()                # a model tag no event carries


def test_confirm_rule():
    rng = np.random.default_rng(3)
    n_streams = 100
    ids = rng.integers(-5, n_streams + 5, 500).astype(np.int32)
    ids[:4] = [-1, n_streams, 0, n_streams - 1]
    scores = rng.random(500, dtype=np.float32)
    scores[::7] = np.nan
    for cutoff in (0.0, 0.25, 0.5, 0.999, -1.0, 2.0):
        got_s, got_c = run_confirm(ids, n_streams, scores, cutoff)
        want_s, want_c = confirm_ref(ids, n_streams, scores, cutoff)
        assert np.array_equal(got_s, want_s, equal_nan=True) and np.array_equal(got_c, want_c)
        listed = (ids >= 0) & (ids < n_streams)
        assert np.array_equal(got_s.view(np.uint32)[listed], scores.view(np.uint32)[listed])     # kept bit for bit
        assert np.isnan(got_s[~listed]).all() and (got_c[~listed] == -1).all()
        assert (got_c[np.isnan(scores)] == -1).all()


def test_confirm_compares_in_double():
    s = np.float32(0.7)                                              # 0.699999988079071 as a double
    d = float(s)
    ids = np.zeros(1, np.int32) + 9
    for cutoff, fires in ((np.nextafter(d, -1.0), True), (d, False), (np.nextafter(d, 2.0), False), (0.7, False), (0.6999999, True)):
        _, c = run_confirm(ids, 10, np.array([s]), float(cutoff))
        assert c[0] == (9 if fires else -1), cutoff
    # a cutoff between the float32 neighbours of the score: only a double comparison tells them apart
    lo = np.nextafter(s, np.float32(0))
    _, c = run_confirm(np.array([1, 2], np.int32), 10, np.array([lo, s]), (float(lo) + d) / 2)
    assert c.tolist() == [-1, 2]


# ---- ABI ------------------------------------------------------------------------------------------------------------------------------
NEW = ("mww_verifier_create", "mww_verifier_destroy", "mww_verifier_info", "mww_verify_streams", "mww_verify_detections")


def test_new_symbols_are_declared_and_exported_with_their_arguments():
    from microwakeword_b200 import _lib, build
    L = _lib.lib()
    assert all(n in _lib.EXPORTS and hasattr(L, n) for n in NEW)
    syms = subprocess.run(["nm", "-D", "--defined-only", build.OUT], capture_output=True, text=True, check=True).stdout
    assert all(re.search(r"\bT %s\b" % n, syms) for n in NEW)
    hdr = open(os.path.join(ROOT, "include", "mww.h")).read()
    flat = re.sub(r"\s+", " ", re.sub(r"/\*.*?\*/", "", hdr, flags=re.S))
    assert ("int mww_verifier_create(const void *model_blob, size_t n_bytes, int device, int slots, const mww_verify_rule *rule, "
            "mww_verifier_t **out);") in flat
    assert "int mww_verifier_info(const mww_verifier_t *v, mww_verifier_desc *out);" in flat
    assert ("int mww_verify_streams(mww_verifier_t *v, mww_t *src, const int32_t *d_ids, int n, float *d_scores, int32_t *d_confirmed, "
            "void *cu_stream);") in flat
    assert ("int mww_verify_detections(mww_verifier_t *v, mww_t *src, mww_detector_t *det, int model, float *d_scores, "
            "int32_t *d_confirmed, void *cu_stream);") in flat
    assert "typedef struct mww_verify_rule { int32_t n_samples, window, ignore_steps, pad; double cutoff; } mww_verify_rule;" in flat
    assert "typedef struct mww_verifier_desc { int32_t slots, steps, device, pad; mww_verify_rule rule; int64_t launches; } mww_verifier_desc;" in flat
    assert [n for n, _ in _lib.MwwVerifyRule._fields_] == ["n_samples", "window", "ignore_steps", "pad", "cutoff"]
    assert ctypes.sizeof(_lib.MwwVerifyRule) == 24 and ctypes.sizeof(_lib.MwwVerifierDesc) == 16 + 24 + 8
    vp, i32 = ctypes.c_void_p, ctypes.c_int
    assert L.mww_verify_streams.argtypes == [vp, vp, vp, i32, vp, vp, vp]
    assert L.mww_verify_detections.argtypes == [vp, vp, vp, i32, vp, vp, vp]


def _rule(n_samples=32000, window=5, ignore=25, cutoff=0.5):
    from microwakeword_b200 import _lib
    return _lib.MwwVerifyRule(n_samples, window, ignore, 0, cutoff)


def test_c_refusals_before_any_device_work():
    """argument refusals come before the device is looked for, so they answer the same with or without a GPU"""
    from microwakeword_b200 import _lib
    L = _lib.lib()
    blob = open(os.path.join(GOLDEN, "okay_nabu_synth_f32.mww"), "rb").read()
    out = ctypes.c_void_p(1)
    for slots, rule, words in ((0, _rule(), b"slots"), (4, _rule(n_samples=479), b"n_samples"), (4, _rule(n_samples=(1 << 22) + 1), b"n_samples"),
                               (4, _rule(window=0), b"window"), (4, _rule(window=33), b"window"), (4, _rule(ignore=-1), b"ignore_steps"),
                               (4, _rule(cutoff=float("nan")), b"cutoff"), (4, _rule(cutoff=float("inf")), b"cutoff")):
        assert L.mww_verifier_create(blob, len(blob), 0, slots, ctypes.byref(rule), ctypes.byref(out)) == -1
        assert words in L.mww_last_error(None) and out.value is None
    assert L.mww_verifier_create(blob, len(blob), 0, 4, None, ctypes.byref(out)) == -1
    assert L.mww_verifier_info(None, None) == -1
    assert L.mww_verify_streams(None, None, None, 0, None, None, None) == -1 and b"verifier" in L.mww_last_error(None)
    assert L.mww_verify_detections(None, None, None, -1, None, None, None) == -1 and b"detector" in L.mww_last_error(None)
    assert L.mww_verifier_destroy(None) == 0


def test_create_without_a_gpu_fails_loudly():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present; the loud-failure path is exercised on GPU-less hosts")
    from microwakeword_b200 import _lib
    from microwakeword_b200.verify import Verifier
    with pytest.raises(_lib.MwwError) as e:
        Verifier(os.path.join(GOLDEN, "okay_nabu_synth_f32.mww"), slots=4, n_samples=32000, cutoff=0.5)
    assert e.value.code == -3 and "no CUDA device" in str(e.value)


# ---- Python ---------------------------------------------------------------------------------------------------------------------------
class NoLib:
    def __getattr__(self, name):
        raise AssertionError("the library was called: %s" % name)


def test_python_create_refusals_before_the_library_is_called(monkeypatch):
    from microwakeword_b200 import _lib
    from microwakeword_b200.verify import Verifier

    def no_lib():
        raise AssertionError("the library was loaded")

    monkeypatch.setattr(_lib, "lib", no_lib)
    model = os.path.join(GOLDEN, "okay_nabu_synth_f32.mww")
    for kw in (dict(slots=0), dict(slots=1.5), dict(slots=True), dict(n_samples=479), dict(n_samples=(1 << 22) + 8), dict(window=0),
               dict(window=33), dict(ignore_steps=-1), dict(cutoff=float("nan")), dict(cutoff=float("-inf")), dict(cutoff="0.5"),
               dict(model=None)):
        args = dict(model=model, slots=4, n_samples=32000, cutoff=0.5)
        args.update(kw)
        with pytest.raises(ValueError):
            Verifier(**args)


def _bare(cls, **attrs):
    o = object.__new__(cls)
    o.__dict__.update(attrs)
    return o


class _Engine:
    def __init__(self, device=0, capacity=32000):
        self.device, self.audio_history_capacity, self._h = device, capacity, None


def test_python_verify_refusals_before_the_library_is_called():
    from microwakeword_b200.detection import MultiModelDetector, StreamDetector
    from microwakeword_b200.verify import Verifier
    v = _bare(Verifier, _L=NoLib(), _v=None, slots=8, n_samples=32000, device=0)
    ids = [0, 1]
    with pytest.raises(ValueError):
        v.verify(_Engine(capacity=0), ids)                               # no audio history
    with pytest.raises(ValueError):
        v.verify(_Engine(capacity=31992), ids)                           # shorter than the verifier reads
    with pytest.raises(ValueError):
        v.verify(_Engine(device=1), ids)                                 # another device
    for bad in (list(range(9)), [0.5], [[0, 1]], np.zeros(3, np.float32)):
        with pytest.raises(ValueError):
            v.verify(_Engine(), bad)                                     # more ids than slots, not integers, not 1-D
    with pytest.raises(ValueError):
        v.verify(_Engine(), ids, model=0)                                # model selects a detector's events only
    plain = _bare(StreamDetector, _L=NoLib(), device=0, capacity=8)
    for m in (1, -1, True, 0.0):
        with pytest.raises(ValueError):
            v.verify(_Engine(), plain, model=m)                          # a plain detector has one model
    with pytest.raises(ValueError):
        v.verify(_Engine(), _bare(StreamDetector, _L=NoLib(), device=0, capacity=9))      # capacity above the slots
    with pytest.raises(ValueError):
        v.verify(_Engine(), _bare(StreamDetector, _L=NoLib(), device=1, capacity=8))      # another device
    multi = _bare(MultiModelDetector, _L=NoLib(), device=0, capacity=8, n_models=3)
    with pytest.raises(ValueError):
        v.verify(_Engine(), multi, model=3)


# ---- build ----------------------------------------------------------------------------------------------------------------------------
def _res_usage(so):
    from microwakeword_b200 import _lib, build
    tool = os.path.join(os.path.dirname(build.NVCC), "cuobjdump")
    if not os.path.exists(tool):
        pytest.skip("cuobjdump is not installed next to nvcc")
    _lib.lib()
    return subprocess.run([tool, "-res-usage", so], capture_output=True, text=True, check=True).stdout


def test_companion_library_holds_exactly_its_two_kernels_without_stack_or_local_memory():
    from microwakeword_b200 import build
    assert os.path.basename(build.VER_OUT) == "libmww_verify.so" and build.VER_SOURCES == ["mww_verify.cu"]
    assert "mww_verify_capi.cu" in build.SOURCES and "mww_verify.cu" not in build.SOURCES
    res = _res_usage(build.VER_OUT)
    found = re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", res)
    names = sorted(n for n, *_ in found)
    assert len(names) == 2 and any("verify_slots_kernel" in n for n in names) and any("verify_confirm_kernel" in n for n in names), res
    assert all(int(stack) == int(local) == 0 for _, _, stack, local in found), found
    flags = [f for f in build.FLAGS if f not in ("-shared", "-cudart", "static")]
    rep = subprocess.run([build.NVCC] + flags + ["-cubin", "-Xptxas", "-v", "-o", os.path.join(_BUILD.name, "verify.cubin"),
                                                 os.path.join(CSRC, "mww_verify.cu")], capture_output=True, text=True, check=True).stderr
    spills = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", rep)
    assert len(spills) == 2 and all(int(a) == int(b) == int(c) == 0 for a, b, c in spills), rep
    # libmww_b200.so holds neither kernel and finds the library next to itself
    main = _res_usage(build.OUT)
    assert "verify_slots_kernel" not in main and "verify_confirm_kernel" not in main
    if shutil.which("readelf"):
        dyn = subprocess.run(["readelf", "-d", build.OUT], capture_output=True, text=True, check=True).stdout
        assert "[libmww_verify.so]" in dyn and "$ORIGIN" in dyn


def test_stale_check_covers_the_companion_library(monkeypatch):
    from microwakeword_b200 import build
    real = os.path.exists
    monkeypatch.setattr(os.path, "exists", lambda p: False if p == build.VER_OUT else real(p))
    assert build._stale()


def test_timing_tool_fails_loudly_without_a_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present; the loud-failure path is exercised on GPU-less hosts")
    tool = os.path.join(ROOT, "tools", "verify_time.py")
    res = subprocess.run([sys.executable, tool, "--rounds", "1"], capture_output=True, text=True)
    assert res.returncode != 0 and "CUDA" in res.stderr
