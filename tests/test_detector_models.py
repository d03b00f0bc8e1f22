"""The multi-model streaming detector (mww_multi_detector_create, MultiModelDetector), the parts that need no GPU: the NumPy
reference (tests/detector_models_ref.py) against K plain detectors (tests/detector_ref.py) when there is no VAD and
against itself over every split of the feature rows into calls; the per-stream body and reset of
microwakeword_b200/csrc/mww_detector_models.h built for the host (tests/emul_detector_models.cc) against that reference,
bit for bit, over random strides, pending rows, splits, windows, NaN, VAD sets and resets, and past the event capacity;
the call-consistency check; the C-ABI's symbols, struct and refusals; the loud failure without a GPU; the register report
of the new kernels and the link of the new library."""

import ctypes
import inspect
import os
import re
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from conftest import ROOT
from detector_models_ref import (MEVENT, OFF, VAD, WAKE, ModelsRef, call_fits, call_steps, feed, same_model_events,
                                 same_model_state)
from detector_ref import DetectorRef, same_events, same_state

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(ROOT, "microwakeword_b200", "csrc")
_BUILD = tempfile.TemporaryDirectory(prefix="mww_detector_models_test_")
_emul = None


def emul():
    global _emul
    if _emul is None:
        so = os.path.join(_BUILD.name, "libemul_detector_models.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "emul_detector_models.cc")], check=True)
        _emul = ctypes.CDLL(so)
        vp, i32, ll = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong
        model_args = [i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]
        _emul.emul_models_update.restype = ll
        _emul.emul_models_update.argtypes = model_args + [vp, vp, vp, vp, vp, vp, i32]
        _emul.emul_models_reset.restype = None
        _emul.emul_models_reset.argtypes = model_args + [vp, i32]
        _emul.emul_call_fits.restype = i32
        _emul.emul_call_fits.argtypes = [i32, vp, vp, vp, vp]
    return _emul


def _i32(v):
    return np.ascontiguousarray(v, np.int32)


def _ptrs(arrays):
    return (ctypes.c_void_p * len(arrays))(*[None if a is None else a.ctypes.data for a in arrays])


class Emulated:
    """the header's body on host state in the device layout; the interface of ModelsRef.  `capacity`: event slots per
    call (None: enough for every step)."""

    def __init__(self, n_streams, roles, windows, cutoffs, cooldowns, strides, streams=None, capacity=None):
        K = len(roles)
        self.n_streams, self.K, self.roles, self.capacity = n_streams, K, list(roles), capacity
        self.windows = [int(w) for w in windows]
        self.streams = [np.arange(n_streams, dtype=np.int32) if streams is None or streams[k] is None else _i32(streams[k]) for k in range(K)]
        self.inv = []
        for s in self.streams:
            if s.size == n_streams:
                self.inv.append(None)
            else:
                inv = np.full(n_streams, -1, np.int32)
                inv[s] = np.arange(s.size)
                self.inv.append(inv)
        self.hist = [np.zeros((max(w - 1, 1), max(s.size, 1)), np.float32) for w, s in zip(self.windows, self.streams)]
        self.seen = [np.zeros(max(s.size, 1), np.int64) for s in self.streams]
        self.flag = [np.zeros(max(s.size, 1), np.int32) for s in self.streams]
        self.arrays = (_i32(roles), _i32(windows), _i32(cooldowns), np.ascontiguousarray(cutoffs, np.float64), _i32(strides),
                       _i32([s.size for s in self.streams]))
        self.count = 0
        self.last_fired = None
        self.reset()

    def _model_args(self):
        r, w, c, cut, s, n = self.arrays
        return [self.n_streams, self.K, r.ctypes.data, w.ctypes.data, c.ctypes.data, cut.ctypes.data, s.ctypes.data, n.ctypes.data,
                _ptrs(self.inv), _ptrs(self.hist), _ptrs(self.seen), _ptrs(self.flag)]

    def reset(self, ids=None):
        a = None if ids is None else _i32(np.asarray(ids).reshape(-1))
        emul().emul_models_reset(*self._model_args(), None if a is None else a.ctypes.data, 0 if a is None else a.size)

    def update(self, probs, n_steps, pending, pitch_pad=0):
        keep = []
        for k in range(self.K):
            if probs[k] is None or self.roles[k] == OFF:
                keep.append(np.zeros((1, 1), np.float32))
                continue
            p = np.asarray(probs[k], np.float32)
            wide = np.full((p.shape[0], p.shape[1] + pitch_pad), 9.0, np.float32)        # past the steps: never read
            wide[:, :p.shape[1]] = p
            keep.append(np.ascontiguousarray(wide) if wide.size else np.zeros((1, 1), np.float32))
        pitch = np.asarray([k.shape[1] for k in keep], np.int64)
        cap = self.capacity or max(1, self.n_streams * max(n_steps) * self.K)
        buf = np.zeros(cap, [("stream", np.int32), ("reserved", np.int32), ("step", np.int64), ("score", np.float32), ("pad", np.int32)])
        fired = np.full(cap, -1, np.int32)
        n, p = _i32(n_steps), _i32(pending)
        got = emul().emul_models_update(*self._model_args(), _ptrs(keep), pitch.ctypes.data, n.ctypes.data, p.ctypes.data,
                                        buf.ctypes.data, fired.ctypes.data, cap)
        assert got >= 0, "the call does not fit"
        self.count = got
        stored = buf[:min(got, cap)]
        assert (stored["pad"] == 0).all()
        self.last_fired = fired
        ev = np.zeros(stored.size, MEVENT)
        ev["stream"], ev["model"], ev["step"], ev["score"] = stored["stream"], stored["reserved"], stored["step"], stored["score"]
        assert np.array_equal(fired[:stored.size], stored["stream"]) and (fired[stored.size:] == -1).all()
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
def _wake_probs(rng, rows, n):
    """uniform, with runs of high values and a NaN now and then"""
    p = rng.random((rows, n)).astype(np.float32)
    for r in range(rows):
        if n > 6 and rng.random() < 0.5:
            at = int(rng.integers(0, n - 5))
            p[r, at:at + 5] = np.float32(0.95)
        if n and rng.random() < 0.2:
            p[r, int(rng.integers(0, n))] = np.nan
    return p


def _vad_probs(rng, rows, n):
    """speech and silence in runs of a few steps, so the flag turns on and off"""
    runs = (rng.random((rows, (n + 3) // 4 + 1)) < 0.55).astype(np.float32)
    p = np.repeat(runs, 4, 1)[:, :n] * 0.9 + 0.05 * rng.random((rows, n)).astype(np.float32)
    if n:
        p[0, n // 2] = np.nan
    return p.astype(np.float32)


def _row_splits(rng, total, count=6):
    """splits of `total` feature rows into calls: one call, 3-row live calls, and random mixtures with 0-row calls and calls
    that end mid-stride"""
    out = [[total], [3] * (total // 3) + ([total % 3] if total % 3 else [])]
    for _ in range(count):
        seq, left = [], total
        while left:
            s = min(int(rng.choice([0, 1, 2, 3, 5, 7, 16, 40])), left)
            seq.append(s)
            left -= s
        out.append(seq)
    return out


def _case(seed, n_streams=45, K=3, vad=True, windows=None, cooldowns=None, sets=True, all_off_but=None):
    """roles, windows, cutoffs, cooldowns, strides, stream sets, starting pending rows, total rows and whole sequences"""
    rng = np.random.default_rng(seed)
    roles = [WAKE] * K
    if vad:
        roles[int(rng.integers(0, K))] = VAD
    if all_off_but is not None:
        roles = [r if k in all_off_but else OFF for k, r in enumerate(roles)]
    # a VAD of a long stride and a long window may never see a full window in a few hundred rows
    windows = windows or [int(rng.choice([1, 2, 5, 9] if roles[k] == VAD else [1, 2, 5, 9, 32])) for k in range(K)]
    cooldowns = cooldowns or [int(rng.choice([0, 1, 3, 25])) for _ in range(K)]
    cutoffs = [float(np.float32(rng.uniform(0.4, 0.7))) for _ in range(K)]
    strides = [int(rng.integers(1, 18)) for _ in range(K)]
    streams = [None] * K
    if sets:
        for k in range(K):
            kind = rng.integers(0, 3 if roles[k] == VAD else 4)     # an empty VAD set would silence every wake word
            streams[k] = (None if kind == 0 else np.flatnonzero(rng.random(n_streams) < 0.6).astype(np.int32) if kind == 1
                          else np.arange(n_streams // 3, n_streams, dtype=np.int32) if kind == 2 else np.zeros(0, np.int32))
    pending0 = [int(rng.integers(0, s)) for s in strides]
    total = int(rng.integers(150, 260))
    seqs = []
    for k in range(K):
        rows = n_streams if streams[k] is None else streams[k].size
        n = (pending0[k] + total) // strides[k]
        seqs.append(None if roles[k] == OFF else (_vad_probs if roles[k] == VAD else _wake_probs)(rng, rows, n))
    return dict(roles=roles, windows=windows, cutoffs=cutoffs, cooldowns=cooldowns, strides=strides, streams=streams,
                pending0=pending0, total=total, seqs=seqs, rng=rng, n_streams=n_streams)


def _make(cls, c, **kw):
    return cls(c["n_streams"], c["roles"], c["windows"], c["cutoffs"], c["cooldowns"], c["strides"], c["streams"], **kw)


# ---- the reference ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(6))
def test_reference_without_a_vad_is_k_plain_detectors(seed):
    c = _case(seed, vad=False)
    rng = c["rng"]
    for split in _row_splits(rng, c["total"], 2):
        ref = _make(ModelsRef, c)
        ev, _ = feed(ref, c["seqs"], c["strides"], c["pending0"], split)
        state = ref.state()
        for k in range(3):
            ids = c["streams"][k] if c["streams"][k] is not None else np.arange(c["n_streams"], dtype=np.int32)
            if ids.size == 0:                                  # a plain detector has at least one row
                assert not (ev["model"] == k).any() and state[k]["seen"].size == 0
                continue
            plain = DetectorRef(ids.size, c["cutoffs"][k], c["windows"][k], c["cooldowns"][k], stream_ids=ids)
            want = plain.update(c["seqs"][k])
            mine = ev[ev["model"] == k]
            assert same_events(mine, want), (seed, k, split)
            assert same_state(state[k], plain.state())


@pytest.mark.parametrize("seed", range(6))
def test_reference_does_not_depend_on_the_split_into_calls(seed):
    c = _case(100 + seed)
    whole = _make(ModelsRef, c)
    want, pend = feed(whole, c["seqs"], c["strides"], c["pending0"], [c["total"]])
    assert want.size > 0
    for split in _row_splits(c["rng"], c["total"]):
        ref = _make(ModelsRef, c)
        got, p = feed(ref, c["seqs"], c["strides"], c["pending0"], split)
        assert p == pend and same_model_events(got, want), split
        assert same_model_state(ref.state(), whole.state())


def test_the_vad_gates_and_order_on_a_shared_row():
    """a hand-made case: stride 1 WAKE (window 1) and stride 2 VAD (window 1); a WAKE step that ends on the row of a VAD step
    sees that step's flag"""
    ref = ModelsRef(1, [WAKE, VAD], [1, 1], [0.5, 0.5], [0, 0], [1, 2])
    wake = np.asarray([[0.9] * 8], np.float32)
    vad = np.asarray([[0.9, 0.1, 0.9, 0.9]], np.float32)
    ev = ref.update([wake, vad], [8, 4], [0, 0])
    # VAD steps end at rows 1, 3, 5, 7: active from row 1 to 2, off for rows 3-4, on from row 5
    assert ev["step"].tolist() == [1, 2, 5, 6, 7]


# ---- the header's body against the reference --------------------------------------------------------------------------------
EMUL_CASES = [
    dict(seed=1), dict(seed=2, vad=False), dict(seed=3, windows=[1, 32, 5], cooldowns=[0, 0, 0]),
    dict(seed=4, windows=[32, 1, 32], cooldowns=[0, 25, 1]), dict(seed=5, K=4), dict(seed=6, sets=False),
    dict(seed=7, n_streams=33, K=2), dict(seed=8, all_off_but=[0, 2]), dict(seed=9, n_streams=64, K=5),
]


@pytest.mark.parametrize("case", EMUL_CASES, ids=[str(c) for c in EMUL_CASES])
def test_emulation_equals_the_reference_for_every_split(case):
    c = _case(**case)
    roles = c["roles"]
    if WAKE not in roles:
        pytest.skip("no WAKE model in this draw")
    for i, split in enumerate(_row_splits(c["rng"], c["total"], 4)):
        # resets in the middle of the sequence: a few global ids (one out of range), then everything
        resets = {len(split) // 3: [0, 5, 7, c["n_streams"] - 1, c["n_streams"] + 3], 2 * len(split) // 3: None} if i % 2 else None
        ref, em = _make(ModelsRef, c), _make(Emulated, c)
        want, _ = feed(ref, c["seqs"], c["strides"], c["pending0"], split, resets)
        got, _ = feed(em, c["seqs"], c["strides"], c["pending0"], split, resets)
        assert same_model_events(got, want), (case, split)
        assert same_model_state(em.state(), ref.state()), (case, split)


def test_pitch_beyond_the_steps_is_not_read():
    c = _case(21)
    ref, em = _make(ModelsRef, c), _make(Emulated, c)
    pending, at = list(c["pending0"]), [0, 0, 0]
    for rows in (4, 30, 0, 9, 60):
        n, after = call_steps(c["strides"], pending, rows)
        probs = [s[:, a:a + m] for s, a, m in zip(c["seqs"], at, n)]
        assert same_model_events(em.update(probs, n, pending, pitch_pad=5), ref.update(probs, n, pending))
        at, pending = [a + m for a, m in zip(at, n)], after
    assert same_model_state(em.state(), ref.state())


def test_events_past_the_capacity_are_counted_and_the_state_advances():
    c = _case(31, n_streams=64, windows=[1, 1, 1], cooldowns=[0, 0, 0], vad=False)
    c["seqs"] = [np.full_like(s, 0.99) for s in c["seqs"]]
    ref, em = _make(ModelsRef, c), _make(Emulated, c, capacity=7)
    pending, at = list(c["pending0"]), [0, 0, 0]
    for rows in (20, 3, 50):
        n, after = call_steps(c["strides"], pending, rows)
        probs = [s[:, a:a + m] for s, a, m in zip(c["seqs"], at, n)]
        want = ref.update(probs, n, pending)
        got = em.update(probs, n, pending)
        assert em.count == want.size > 7 and got.size == 7
        keys = {(int(e["stream"]), int(e["model"]), int(e["step"])) for e in want}
        assert all((int(e["stream"]), int(e["model"]), int(e["step"])) in keys for e in got)
        at, pending = [a + m for a, m in zip(at, n)], after
    assert same_model_state(em.state(), ref.state())


def test_call_consistency_check():
    rng = np.random.default_rng(5)
    seen = {True: 0, False: 0}
    for _ in range(3000):
        K = int(rng.integers(1, 5))
        roles = [int(rng.choice([OFF, WAKE, WAKE, VAD])) for _ in range(K)]
        if all(r == OFF for r in roles):
            roles[0] = WAKE
        strides = [int(rng.integers(1, 18)) for _ in range(K)]
        pending = [int(rng.integers(0, s)) for s in strides]
        if rng.random() < 0.5:                               # a real call, then perhaps one number off
            n, _ = call_steps(strides, pending, int(rng.integers(0, 60)))
            if rng.random() < 0.5:
                k = int(rng.integers(0, K))
                if rng.random() < 0.5:
                    n[k] += int(rng.choice([-1, 1]))
                else:
                    pending[k] = int(rng.integers(-1, strides[k] + 1))
        else:
            n = [int(rng.integers(0, 6)) for _ in range(K)]
        want = call_fits(roles, strides, n, pending)
        args = [_i32(v) for v in (roles, strides, n, pending)]              # kept alive across the call
        got = emul().emul_call_fits(K, *[a.ctypes.data for a in args])
        assert bool(got) == want, (roles, strides, n, pending)
        seen[want] += 1
    assert min(seen.values()) > 300


# ---- C-ABI -----------------------------------------------------------------------------------------------------------------------
def test_struct_and_the_rule_in_the_header():
    from microwakeword_b200 import _lib
    assert ctypes.sizeof(_lib.MwwDetectRule) == emul().emul_sizeof_rule() == 24
    hdr = open(os.path.join(ROOT, "include", "mww.h")).read()
    assert "typedef struct mww_detect_rule { int32_t role, window, cooldown_slices, pad; double cutoff; } mww_detect_rule;" in hdr
    for line in ("e_k(j) = (j + 1) s_k - p_k - 1", "When a VAD step and a WAKE step end on the same", "A stream that is not in S_v is never active",
                 "the row fires iff cooldown == 0 && (double)avg > cutoff_k && gate", "reserved = the model index k"):
        assert line in re.sub(r"\s*\n\s*\*\s*", " ", hdr), line
    for name, v in (("MWW_DETECT_OFF", 0), ("MWW_DETECT_WAKE", 1), ("MWW_DETECT_VAD", 2)):
        assert "#define %s %d" % (name, v) in hdr and getattr(_lib, name) == v


PLAIN = ("mww_detector_create", "mww_detector_destroy", "mww_detector_update", "mww_detector_drain", "mww_detector_buffers",
         "mww_detector_reset", "mww_detector_reset_device", "mww_detector_get_state", "mww_detector_set_state")
MULTI = ("mww_multi_detector_create", "mww_multi_detector_update", "mww_multi_detector_get_state", "mww_multi_detector_set_state")


def test_multi_detector_symbols_are_exported():
    """the multi-model detector's four calls, beside (not among) the plain detector's nine"""
    from microwakeword_b200 import _lib
    L = _lib.lib()
    assert sorted(n for n in _lib.EXPORTS if n.startswith("mww_multi_detector_")) == sorted(MULTI)
    assert sorted(n for n in _lib.EXPORTS if n.startswith("mww_detector_")) == sorted(PLAIN)
    for n in PLAIN + MULTI:
        assert hasattr(L, n)


def _rules(*roles):
    from microwakeword_b200 import _lib
    return (_lib.MwwDetectRule * len(roles))(*[_lib.MwwDetectRule(r, 5, 25, 0, 0.5) for r in roles])


def test_arguments_refused_before_any_device_work():
    from microwakeword_b200 import _lib
    L = _lib.lib()
    d = ctypes.c_void_p()
    assert L.mww_multi_detector_create(None, _rules(WAKE), 0, ctypes.byref(d)) == -1 and b"capacity" in L.mww_last_error(None)
    assert L.mww_multi_detector_create(None, None, 16, ctypes.byref(d)) == -1 and b"rules" in L.mww_last_error(None)
    assert L.mww_multi_detector_create(None, _rules(WAKE), 16, None) == -1
    z = (ctypes.c_int * 1)(0)
    pz = (ctypes.c_longlong * 1)(0)
    assert L.mww_multi_detector_update(None, None, pz, z, z, None) == -1
    assert L.mww_multi_detector_get_state(None, 0, None, None, None) == -1
    assert L.mww_multi_detector_set_state(None, 0, None, None, None) == -1
    assert not d.value


def test_no_cpu_fallback_without_a_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present; the loud-failure path is exercised on GPU-less hosts")
    from microwakeword_b200 import _lib
    L = _lib.lib()
    d = ctypes.c_void_p()
    assert L.mww_multi_detector_create(None, _rules(WAKE, VAD), 16, ctypes.byref(d)) == -3
    assert b"no CUDA device" in L.mww_last_error(None) and not d.value
    tool = os.path.join(ROOT, "tools", "detector_models_time.py")
    res = subprocess.run([sys.executable, tool, "--streams", "64"], capture_output=True, text=True)
    assert res.returncode != 0 and "CUDA" in res.stderr


# ---- build -------------------------------------------------------------------------------------------------------------------
def test_models_detector_kernels_do_not_spill():
    from microwakeword_b200 import build
    if not os.path.exists(build.NVCC):
        pytest.skip("nvcc is not installed")
    flags = [f for f in build.FLAGS if f not in ("-shared", "-cudart", "static")]
    res = subprocess.run([build.NVCC] + flags + ["-cubin", "-Xptxas", "-v", "-o", os.path.join(_BUILD.name, "detector_models.cubin"),
                                                  os.path.join(CSRC, "mww_detector_models.cu")], capture_output=True, text=True, check=True)
    reports = re.findall(r"Function properties for (\S+)\s+(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", res.stderr)
    names = sorted(name for name, *_ in reports)
    assert len(names) == 2 and any("detector_models_update_kernel" in n for n in names) and any("detector_models_reset_kernel" in n for n in names), res.stderr
    assert all(int(stack) == int(st) == int(ld) == 0 for _, stack, st, ld in reports), reports


def test_main_library_links_the_models_detector_library():
    from microwakeword_b200 import build
    assert os.path.basename(build.MD_OUT) == "libmww_detector_models.so" and build.MD_SOURCES == ["mww_detector_models.cu"]
    assert "MD_OUT" in inspect.getsource(build._stale)
    from microwakeword_b200 import _lib
    _lib.lib()
    assert os.path.exists(build.MD_OUT)
    import shutil
    if shutil.which("readelf"):
        dyn = subprocess.run(["readelf", "-d", build.OUT], capture_output=True, text=True, check=True)
        assert "[libmww_detector_models.so]" in dyn.stdout and "$ORIGIN" in dyn.stdout
