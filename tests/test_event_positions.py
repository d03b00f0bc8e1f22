"""Event positions (include/mww.h, "event positions"), the parts that need no GPU: the timed detectors' bodies, the history
read that ends at given positions and the verifier slots that end at their events, built with g++ from
microwakeword_b200/csrc/mww_event_positions.h by tests/emul_event_positions.cc and checked against NumPy:

- events fired by tests/detector_ref.py / tests/detector_models_ref.py over random probabilities, every split of a sequence
  into calls and resets between calls, each placed with the clock of the call it fired in (the thread form, the warp form lane
  by lane, and the models body with a VAD, whose positions are checked against the endpointer's formula);
- the read against a NumPy ring: ends inside, straddling and outside [S - C, S), negative ends and -1 ids, in the vector and
  the scalar form; the slots against the rule: e clamped at S and the expiry condition;
- every pre-existing kernel's instructions against tests/golden/sass_kernels_before_event_positions.json (the parent's
  build), each library's kernel count, the new library's kernels without stack or local memory, its link and stale check;
- the new symbols with their argument types, no new mww_detector_* / mww_multi_detector_* export, and the refusals that need
  no detector."""

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

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from detector_models_ref import OFF, VAD, WAKE, ModelsRef, call_steps  # noqa: E402
from detector_ref import DetectorRef  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(ROOT, "microwakeword_b200", "csrc")
_BUILD = tempfile.TemporaryDirectory(prefix="mww_event_positions_test_")
_emul = []
EVENT = np.dtype([("stream", np.int32), ("reserved", np.int32), ("step", np.int64), ("score", np.float32), ("pad", np.int32)])
vp, i32, ll, dbl = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_double


def emul():
    if not _emul:
        so = os.path.join(_BUILD.name, "libemul_event_positions.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "emul_event_positions.cc")], check=True)
        L = ctypes.CDLL(so)
        for fn in (L.emul_timed_thread, L.emul_timed_warp):
            fn.restype = ll
            fn.argtypes = [i32, dbl, i32, vp, vp, vp, vp, i32, i32, ll, ll, ll, vp, vp, i32]
        L.emul_call_rows.restype = ll
        L.emul_call_rows.argtypes = [i32, vp, vp, vp, vp, vp]
        L.emul_timed_models.restype = ll
        L.emul_timed_models.argtypes = [i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, ll, i32, vp, vp, i32]
        L.emul_read_at.restype = None
        L.emul_read_at.argtypes = [vp, i32, ll, vp, vp, i32, i32, i32, vp, ll, i32]
        L.emul_slots_at.restype = None
        L.emul_slots_at.argtypes = [ll, i32, vp, vp, i32, ll, ll, i32, i32, vp, vp]
        _emul.append(L)
    return _emul[0]


def _ptr(a):
    return a.ctypes.data


# ---- the plain detector ------------------------------------------------------------------------------------------------------------
def splits(total, rng, n=6):
    """every split of `total` steps into two calls, and some random splits into many"""
    out = [[total]] + [[a, total - a] for a in range(1, total)]
    for _ in range(n):
        cuts = np.sort(rng.choice(np.arange(1, total), size=rng.integers(2, 8), replace=False))
        out.append(list(np.diff(np.concatenate([[0], cuts, [total]]))))
    return out


def run_plain(form, probs, calls, window, cutoff, cooldown, clocks, resets):
    R = probs.shape[0]
    hist = np.zeros((R, window - 1), np.float32)
    seen = np.zeros(R, np.int64)
    cd = np.full(R, cooldown, np.int32)
    fn = emul().emul_timed_warp if form == "warp" else emul().emul_timed_thread
    evs, poss, at = [], [], 0
    for c, n in enumerate(calls):
        for r in resets.get(c, []):
            hist[r], seen[r], cd[r] = 0, 0, cooldown
        p = np.ascontiguousarray(probs[:, at:at + n])
        ev, pos = np.zeros(R * max(n, 1), EVENT), np.zeros(R * max(n, 1), np.int64)
        last_end, step = clocks[c]
        got = fn(window, cutoff, cooldown, _ptr(hist), _ptr(seen), _ptr(cd), _ptr(p), R, n, n, last_end, step, _ptr(ev), _ptr(pos), ev.size)
        evs.append(ev[:got])
        poss.append(pos[:got])
        at += n
    return np.concatenate(evs), np.concatenate(poss)


def ref_plain(probs, calls, window, cutoff, cooldown, clocks, resets):
    ref = DetectorRef(probs.shape[0], cutoff, window, cooldown)
    evs, poss, at = [], [], 0
    for c, n in enumerate(calls):
        if c in resets:
            ref.reset(resets[c])
        before = ref.seen.copy()
        ev = ref.update(probs[:, at:at + n])
        t = ev["step"] - before[ev["stream"]]
        last_end, step = clocks[c]
        evs.append(ev)
        poss.append(last_end - (n - 1 - t) * step)
        at += n
    return np.concatenate(evs), np.concatenate(poss)


def same_timed(a, pa, b, pb):
    """the same (stream, step, score bits, position) set"""
    ka = sorted(zip(a["stream"].tolist(), a["step"].tolist(), a["score"].view(np.uint32).tolist(), pa.tolist()))
    kb = sorted(zip(b["stream"].tolist(), b["step"].tolist(), b["score"].view(np.uint32).tolist(), pb.tolist()))
    return ka == kb


@pytest.mark.parametrize("form,total", [("thread", 40), ("warp", 110)])
def test_plain_bodies_place_each_event_with_its_call_clock(form, total):
    rng = np.random.default_rng(1 if form == "thread" else 2)
    R, window, cooldown = 24, 5, 7
    probs = rng.random((R, total), dtype=np.float32)
    probs[:, ::13] = np.nan
    fired = 0
    for i, calls in enumerate(splits(total, rng)):
        if form == "warp" and i % 9:
            continue
        clocks = [(int(rng.integers(-5000, 10 ** 9)), int(rng.integers(1, 2000))) for _ in calls]
        resets = {c: list(rng.choice(R, 3, replace=False)) for c in range(1, len(calls)) if rng.random() < 0.4}
        got = run_plain(form, probs, calls, window, 0.6, cooldown, clocks, resets)
        want = ref_plain(probs, calls, window, 0.6, cooldown, clocks, resets)
        assert same_timed(*got, *want), (form, calls)
        fired += want[0].size
    assert fired > 100


# ---- the models detector ------------------------------------------------------------------------------------------------------------
def endpoint_position(row_end, hop, g, stride, n, j):
    """mww_endpoint.h's endpoint_position with S - b = row_end"""
    return row_end - hop * (g + (n - 1 - j) * stride)


def test_models_body_places_each_event_with_the_endpointer_formula():
    rng = np.random.default_rng(3)
    S, hop = 40, 160
    roles, windows, cooldowns, strides = [WAKE, OFF, WAKE, VAD], [5, 3, 4, 3], [6, 0, 9, 0], [3, 1, 2, 1]
    cut = [0.55, 0.0, 0.6, 0.45]
    rows_total = 150
    seqs = [rng.random((S, rows_total), dtype=np.float32) if r != OFF else None for r in roles]
    fired = 0
    for trial in range(8):
        row_calls = [int(x) for x in rng.integers(0, 9, size=25)]
        hist = [np.zeros((max(w - 1, 1), S), np.float32) for w in windows]
        seen = [np.zeros(S, np.int64) for _ in roles]
        flag = [np.full(S, cooldowns[k] if roles[k] == WAKE else 0, np.int32) for k in range(4)]
        ref = ModelsRef(S, roles, windows, cut, cooldowns, strides)
        pending, at, row_end = [0, 0, 0, 0], [0] * 4, int(rng.integers(0, 10 ** 6))
        got_all, want_all = [], []
        for c, R in enumerate(row_calls):
            if trial % 2 and c % 7 == 3:                   # a reset between calls, of the same streams on both sides
                ids = [int(i) for i in rng.choice(S, 4, replace=False)]
                ref.reset(ids)
                for k in range(4):
                    if roles[k] == OFF:
                        continue
                    for i in ids:
                        hist[k][:, i], seen[k][i], flag[k][i] = 0, 0, cooldowns[k] if roles[k] == WAKE else 0
            n, after = call_steps(strides, pending, R)
            row_end += R * hop
            probs = [np.ascontiguousarray(s[:, a:a + m]) if s is not None else np.zeros((S, 1), np.float32) for s, a, m in zip(seqs, at, n)]
            before = [s.copy() for s in ref.seen]
            want = ref.update([p if r != OFF else None for p, r in zip(probs, roles)], n, pending)
            j = want["step"] - np.array([before[k][s] for k, s in zip(want["model"], want["stream"])], np.int64)
            wpos = np.array([endpoint_position(row_end, hop, after[k], strides[k], n[k], jj) for k, jj in zip(want["model"], j)], np.int64)
            cap = 4096
            ev, pos = np.zeros(cap, EVENT), np.zeros(cap, np.int64)
            keep = dict(roles=np.asarray(roles, np.int32), windows=np.asarray(windows, np.int32), cooldowns=np.asarray(cooldowns, np.int32),
                        cut=np.asarray(cut, np.float64), strides=np.asarray(strides, np.int32), n=np.asarray(n, np.int32),
                        pending=np.asarray(pending, np.int32), after=np.asarray(after, np.int32),
                        pitch=np.asarray([max(p.shape[1], 1) for p in probs], np.int64))
            ptrs = lambda xs: (vp * len(xs))(*[_ptr(x) for x in xs])      # noqa: E731
            got = emul().emul_timed_models(S, 4, _ptr(keep["roles"]), _ptr(keep["windows"]), _ptr(keep["cooldowns"]), _ptr(keep["cut"]),
                                           _ptr(keep["strides"]), ptrs(hist), ptrs(seen), ptrs(flag), ptrs(probs), _ptr(keep["pitch"]),
                                           _ptr(keep["n"]), _ptr(keep["pending"]), _ptr(keep["after"]), row_end, hop, _ptr(ev), _ptr(pos), cap)
            assert got >= 0
            g = ev[:got]
            got_all.append((g["stream"], g["reserved"], g["step"], g["score"].view(np.uint32), pos[:got]))
            want_all.append((want["stream"], want["model"], want["step"], want["score"].view(np.uint32), wpos))
            at = [a + m for a, m in zip(at, n)]
            pending = after
        key = lambda parts: sorted(zip(*[np.concatenate(p).tolist() for p in zip(*parts)]))    # noqa: E731
        assert key(got_all) == key(want_all), trial
        fired += sum(w[0].size for w in want_all)
    assert fired > 50


def _rows(K, roles, strides, n, pending, after):
    a = [np.asarray(x, np.int32) for x in (roles, strides, n, pending, after)]
    return emul().emul_call_rows(K, *[_ptr(x) for x in a])


def test_call_rows_need_the_pending_rows_after_the_call():
    for R in range(0, 20):
        for p0 in range(3):
            for p1 in range(2):
                n, after = call_steps([3, 2], [p0, p1], R)
                assert _rows(2, [WAKE, WAKE], [3, 2], n, [p0, p1], after) == R
    # one stride-3 model, one step: R is 3, 4 or 5 from n and p alone; the pending rows after fix it, and a wrong one is refused
    for g, R in ((0, 3), (1, 4), (2, 5)):
        assert _rows(1, [WAKE], [3], [1], [0], [g]) == R
    assert _rows(1, [WAKE], [3], [1], [0], [3]) == -1
    n, after = call_steps([3, 2], [0, 0], 7)
    after[1] = (after[1] + 1) % 2                          # the two models disagree on R
    assert _rows(2, [WAKE, WAKE], [3, 2], n, [0, 0], after) == -1
    assert _rows(2, [WAKE, OFF], [3, 1], [1, 0], [0, 0], [2, 0]) == 5      # an OFF model does not take part


# ---- the read and the slots ---------------------------------------------------------------------------------------------------------
def ring_model(full, C, seen, ids, ends, n, n_streams):
    """row i: axis positions [end - n, end) of stream id from the whole audio `full`, zeros outside [seen - C, seen), outside
    [0, seen) (never appended) and for ids outside [0, n_streams)"""
    out = np.zeros((len(ids), n), np.int16)
    for r, (s, e) in enumerate(zip(ids, ends)):
        if not 0 <= s < n_streams:
            continue
        for k in range(n):
            t = e - n + k
            if max(seen - C, 0) <= t < seen:
                out[r, k] = full[s, t]
    return out


@pytest.mark.parametrize("C,seen", [(64, 40), (64, 64), (64, 1000), (96, 777)])
def test_read_at_is_the_ring_rule(C, seen):
    rng = np.random.default_rng(C + seen)
    n_streams = 5
    full = rng.integers(-30000, 30000, size=(n_streams, seen), dtype=np.int16)
    ring = np.zeros((n_streams, C), np.int16)
    for t in range(max(0, seen - C), seen):
        ring[:, t % C] = full[:, t]
    ids = np.asarray([0, 1, 2, -1, 4, 3, 7, 2, 1, 0], np.int32)
    ends = np.asarray([seen, seen - 5, seen - C + 16, seen, seen + 40, seen - C - 3, seen, -1, seen - 8, 24], np.int64)
    for n in (0, 8, 16, 24, 13):
        for vec in ((0, 1) if n % 8 == 0 else (0,)):
            stride = max(n, 8) + 8
            out = np.full((ids.size, stride), 99, np.int16)
            emul().emul_read_at(_ptr(ring), C, seen, _ptr(ids), _ptr(ends), ids.size, n_streams, n, _ptr(out), stride, vec)
            assert np.array_equal(out[:, :n], ring_model(full, C, seen, ids, ends, n, n_streams)), (n, vec)
            assert (out[:, n:] == 99).all()                    # nothing past n_samples is written


def test_slots_at_clamp_and_expiry():
    cap, C, N = 12, 1000, 400
    S = 5000
    ev = np.zeros(cap, EVENT)
    ev["stream"] = np.arange(cap) + 100
    ev["reserved"] = np.arange(cap) % 2
    pos = np.asarray([S - 10, S - 300, S - 599, S - 600, S - 601, S, S - 1000, -1, 4000, 4600, 4599, 4601], np.int64)
    for count in (0, 1, 7, cap, cap + 5):
        for model in (-1, 0, 1):
            for post in (0, 1, 200, 2 ** 22):
                ids, ends = np.zeros(cap, np.int32), np.zeros(cap, np.int64)
                emul().emul_slots_at(count, cap, _ptr(ev), _ptr(pos), model, post, S, C, N, _ptr(ids), _ptr(ends))
                for i in range(cap):
                    used = i < min(count, cap) and (model < 0 or ev["reserved"][i] == model)
                    e = min(int(pos[i]) + post, S)
                    ok = used and e - N >= S - C
                    assert ids[i] == (ev["stream"][i] if ok else -1) and ends[i] == (e if ok else -1), (count, model, post, i)


# ---- build, ABI and refusals ----------------------------------------------------------------------------------------------------------
NEW = ("mww_time_detector_events", "mww_update_detector_at", "mww_update_multi_detector_at", "mww_get_detector_positions",
       "mww_drain_detector_at", "mww_read_audio_history_at", "mww_verify_detections_at")


def test_new_symbols_are_declared_and_exported_with_their_arguments():
    from microwakeword_b200 import _lib, build
    L = _lib.lib()
    assert all(n in _lib.EXPORTS and hasattr(L, n) for n in NEW)
    assert not any(n.startswith(("mww_detector_", "mww_multi_detector_")) for n in NEW)
    syms = subprocess.run(["nm", "-D", "--defined-only", build.OUT], capture_output=True, text=True, check=True).stdout
    assert all(re.search(r"\bT %s\b" % n, syms) for n in NEW)
    hdr = re.sub(r"\s+", " ", open(os.path.join(ROOT, "include", "mww.h")).read())
    sigs = {"mww_time_detector_events": "mww_detector_t *d",
            "mww_update_detector_at": "mww_detector_t *d, const float *d_probs, int n_steps, long long pitch, long long last_end, long long step_samples, void *cu_stream",
            "mww_update_multi_detector_at": "mww_detector_t *d, const float *const *d_probs, const long long *pitch, const int *n_steps, "
                                            "const int *pending_before, const int *pending_after, long long row_end, void *cu_stream",
            "mww_get_detector_positions": "mww_detector_t *d, const int64_t **d_positions",
            "mww_drain_detector_at": "mww_detector_t *d, mww_event *h_events, int64_t *h_positions, int max_events, long long *n_events, void *cu_stream",
            "mww_read_audio_history_at": "mww_t *h, const int32_t *d_ids, const long long *d_ends, int n, int n_samples, int16_t *d_out, "
                                         "long long out_stride, void *cu_stream",
            "mww_verify_detections_at": "mww_verifier_t *v, mww_t *src, mww_detector_t *det, int model, long long post, float *d_scores, "
                                        "int32_t *d_confirmed, void *cu_stream"}
    for name, args in sigs.items():
        assert "int %s(%s);" % (name, args) in hdr, name
    want = {"mww_update_detector_at": [vp, vp, i32, ll, ll, ll, vp], "mww_update_multi_detector_at": [vp, vp, vp, vp, vp, vp, ll, vp],
            "mww_read_audio_history_at": [vp, vp, vp, i32, i32, vp, ll, vp], "mww_verify_detections_at": [vp, vp, vp, i32, ll, vp, vp, vp]}
    for name, args in want.items():
        assert getattr(L, name).argtypes == args, name


def test_null_objects_are_refused_without_device_work():
    from microwakeword_b200 import _lib
    L = _lib.lib()
    n = ctypes.c_longlong(0)
    assert L.mww_time_detector_events(None) == -1 and b"NULL" in L.mww_last_error(None)
    assert L.mww_update_detector_at(None, None, 0, 0, 0, 1, None) == -1
    assert L.mww_update_multi_detector_at(None, None, None, None, None, None, 0, None) == -1
    assert L.mww_get_detector_positions(None, ctypes.byref(vp())) == -1
    assert L.mww_drain_detector_at(None, None, None, 0, ctypes.byref(n), None) == -1
    assert L.mww_verify_detections_at(None, None, None, 0, -1, None, None, None) == -1 and b"post" in L.mww_last_error(None)
    assert L.mww_verify_detections_at(None, None, None, 0, 2 ** 22 + 1, None, None, None) == -1
    assert L.mww_read_audio_history_at(None, None, None, 0, 0, None, 0, None) != 0


class _Bare:
    pass


def test_python_refusals_before_the_library_is_called():
    from microwakeword_b200.detection import StreamDetector
    from microwakeword_b200.verify import Verifier
    ver = Verifier.__new__(Verifier)
    ver.device, ver.n_samples, ver.slots = 0, 32000, 16
    det = StreamDetector.__new__(StreamDetector)
    det.timed = False
    with pytest.raises(ValueError, match="timed detector"):
        ver.verify(_Bare(), det, at_event=True)
    with pytest.raises(ValueError, match="timed detector"):
        ver.verify(_Bare(), [0, 1], at_event=True)
    det.timed = True
    for post in (-1, 2 ** 22 + 1, 1.5, True):
        with pytest.raises(ValueError, match="post"):
            ver.verify(_Bare(), det, at_event=True, post=post)
    with pytest.raises(ValueError, match="at_event"):
        ver.verify(_Bare(), det, post=5)
    det.n_rows, det.device = 1, 0
    with pytest.raises(ValueError):
        StreamDetector.update(det, _Bare())                    # not a CUDA tensor: refused before anything else


def _cuobjdump():
    from microwakeword_b200 import _lib, build
    tool = os.path.join(os.path.dirname(build.NVCC), "cuobjdump")
    if not os.path.exists(tool):
        pytest.skip("cuobjdump is not installed next to nvcc")
    _lib.lib()
    return tool


def _sass_hashes(so):
    """kernel -> sha256 of its instruction words, anonymous-namespace ids normalised as the fixture has them"""
    text = subprocess.run([_cuobjdump(), "-sass", so], capture_output=True, text=True, check=True).stdout
    words, name = {}, None
    for line in text.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = re.sub(r"_GLOBAL__N__[0-9a-f]+_\d+_\w+?_[0-9a-f]{8}", "_GLOBAL__N_", m.group(1))
            words[name] = []
        elif name:
            words[name] += re.findall(r"/\* (0x[0-9a-f]{16}) \*/", line)
    return {n: hashlib.sha256(" ".join(w).encode()).hexdigest() for n, w in words.items()}


def test_every_existing_kernel_keeps_its_instructions():
    from microwakeword_b200 import build
    before = json.load(open(os.path.join(GOLDEN, "sass_kernels_before_event_positions.json")))
    libs = [k for k in before if k != "_comment"]
    assert len(libs) == 12
    for lib in libs:
        got = _sass_hashes(os.path.join(os.path.dirname(build.OUT), lib))
        assert got == before[lib], lib


def test_companion_library_holds_exactly_its_kernels_without_stack_or_local_memory(monkeypatch):
    from microwakeword_b200 import build
    assert os.path.basename(build.EVP_OUT) == "libmww_event_positions.so" and build.EVP_SOURCES == ["mww_event_positions.cu"]
    res = subprocess.run([_cuobjdump(), "-res-usage", build.EVP_OUT], capture_output=True, text=True, check=True).stdout
    found = re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", res)
    names = [n for n, *_ in found]
    assert len(names) == 8, res
    assert sum("detector_update_at_kernel" in n for n in names) == 4
    assert sum("detector_models_update_at_kernel" in n for n in names) == 2
    assert sum("history_read_at_kernel" in n for n in names) == 1 and sum("verify_slots_at_kernel" in n for n in names) == 1
    assert all(int(stack) == int(local) == 0 for _, _, stack, local in found), found
    flags = [f for f in build.FLAGS if f not in ("-shared", "-cudart", "static")]
    rep = subprocess.run([build.NVCC] + flags + ["-cubin", "-Xptxas", "-v", "-o", os.path.join(_BUILD.name, "evp.cubin"),
                                                 os.path.join(CSRC, "mww_event_positions.cu")], capture_output=True, text=True, check=True).stderr
    spills = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", rep)
    assert len(spills) == 8 and all(int(a) == int(b) == int(c) == 0 for a, b, c in spills), rep
    if shutil.which("readelf"):
        dyn = subprocess.run(["readelf", "-d", build.OUT], capture_output=True, text=True, check=True).stdout
        assert "[libmww_event_positions.so]" in dyn and "$ORIGIN" in dyn
    real = os.path.exists
    monkeypatch.setattr(build.os.path, "exists", lambda p: p != build.EVP_OUT and real(p))
    assert build._stale()
