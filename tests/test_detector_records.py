"""Detector records (mww_export_detector_rows / mww_import_detector_rows; StreamDetector.export_rows / import_rows and
MultiModelDetector.export_streams / import_streams), the parts that need no GPU: the record layout against sizes worked out
by hand, and the pack and unpack kernels' per-word bodies (microwakeword_b200/csrc/mww_detector_records.h, built with g++ in
a temporary directory by tests/emul_detector_records.cc) against a NumPy model of the rule in include/mww.h, for 1, 3 and 64
models, windows 1, 5 and 32, WAKE, VAD and OFF roles, and imports into detectors with other row counts and stream sets
(taken, fresh and ignored slots; unlisted rows untouched); each layout mismatch and its field; the new symbols and their
argument lists; the Python refusals and a save / load round trip; the companion library's link, kernels and registers; the
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

from conftest import ROOT

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(ROOT, "microwakeword_b200", "csrc")
_BUILD = tempfile.TemporaryDirectory(prefix="mww_detector_records_test_")
_emul = None

OFF, WAKE, VAD = 0, 1, 2


def emul():
    global _emul
    if _emul is None:
        so = os.path.join(_BUILD.name, "libemul_detector_records.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "emul_detector_records.cc")], check=True)
        _emul = ctypes.CDLL(so)
        vp, i32 = ctypes.c_void_p, ctypes.c_int
        _emul.emul_detrec_layout.restype = None
        _emul.emul_detrec_layout.argtypes = [vp, vp, i32, vp]
        for fn in (_emul.emul_detrec_pack, _emul.emul_detrec_unpack):
            fn.restype = i32
            fn.argtypes = [i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, vp]
        _emul.emul_detrec_mismatch.restype = i32
        _emul.emul_detrec_mismatch.argtypes = [vp, vp, ctypes.POINTER(i32), ctypes.c_char_p, i32]
    return _emul


def _i32(v):
    return np.ascontiguousarray(v, np.int32)


def _ptrs(arrays):
    return (ctypes.c_void_p * len(arrays))(*[None if a is None else a.ctypes.data for a in arrays])


def layout(roles, windows):
    K = len(roles)
    out = np.zeros(1 + 2 * K, np.int64)
    r, w = _i32(roles), _i32(windows)
    emul().emul_detrec_layout(r.ctypes.data, w.ctypes.data, K, out.ctypes.data)
    return int(out[0]), out[1:1 + K].tolist(), out[1 + K:].tolist()


# ---- a detector's state in the device layout, and the NumPy model of the rule ------------------------------------------------
class Det:
    """host state of a detector as the kernels see it: per model hist [window - 1][n_rows], seen, flag, and the inverse map
    of its stream set (None: every id, row = id).  A plain detector is one WAKE model over n_ids rows."""

    def __init__(self, n_ids, roles, windows, cooldowns, streams, rng):
        self.n_ids, self.roles, self.windows, self.cooldowns = n_ids, list(roles), list(windows), list(cooldowns)
        self.K = len(roles)
        self.streams = [np.arange(n_ids, dtype=np.int32) if s is None else _i32(s) for s in streams]
        self.inv, self.lookup = [], []
        for s in self.streams:
            inv = np.full(n_ids, -1, np.int32)
            inv[s] = np.arange(s.size)
            self.lookup.append(inv)
            self.inv.append(None if s.size == n_ids else inv)
        # arbitrary bytes everywhere, so that a word written where it should not be shows
        self.hist = [rng.standard_normal((max(w - 1, 1), max(s.size, 1))).astype(np.float32) for w, s in zip(self.windows, self.streams)]
        self.seen = [rng.integers(0, 1 << 40, max(s.size, 1)).astype(np.int64) for s in self.streams]
        self.flag = [rng.integers(0, 30, max(s.size, 1)).astype(np.int32) for s in self.streams]

    def args(self):
        n_rows = _i32([s.size for s in self.streams])
        keep = (_i32(self.roles), _i32(self.windows), _i32(self.cooldowns), n_rows)
        return keep, [self.K] + [a.ctypes.data for a in keep] + [_ptrs(self.inv), _ptrs(self.hist), _ptrs(self.seen), _ptrs(self.flag)]

    def pack(self, ids):
        ids = _i32(ids)
        rb, _, _ = layout(self.roles, [w if r != OFF else 1 for r, w in zip(self.roles, self.windows)])
        rec = np.full((ids.size, rb // 4), 0xA5A5A5A5, np.uint32)
        keep, a = self.args()
        assert emul().emul_detrec_pack(*a, ids.ctypes.data, ids.size, rec.ctypes.data) == rb // 4
        return rec.view(np.uint8).reshape(ids.size, rb)

    def unpack(self, ids, rec):
        ids, rec = _i32(ids), np.ascontiguousarray(rec)
        keep, a = self.args()
        emul().emul_detrec_unpack(*a, ids.ctypes.data, ids.size, rec.ctypes.data)

    def snapshot(self):
        return [(h.copy(), s.copy(), f.copy()) for h, s, f in zip(self.hist, self.seen, self.flag)]


def model_layout(roles, windows):
    """(record_bytes, [(hist_off, tail_off) or None per model]) from the rule in include/mww.h"""
    pad = lambda b: (b + 15) // 16 * 16
    off, slots = 16, []
    for r, w in zip(roles, windows):
        if r == OFF:
            slots.append(None)
            continue
        h = off
        off += pad(4 * (w - 1))
        slots.append((h, off))
        off += 16
    return off, slots


def model_pack(det, ids):
    """the records the rule describes, byte by byte"""
    rb, slots = model_layout(det.roles, det.windows)
    out = np.zeros((len(ids), rb), np.uint8)
    for j, i in enumerate(ids):
        mask = 0
        for k, sl in enumerate(slots):
            if sl is None:
                continue
            row = det.lookup[k][i]
            if row < 0:
                continue
            mask |= 1 << k
            h, t = sl
            w = det.windows[k]
            out[j, h:h + 4 * (w - 1)] = det.hist[k][:w - 1, row].astype("<f4").view(np.uint8)
            out[j, t:t + 8] = np.asarray([det.seen[k][row]], "<i8").view(np.uint8)
            out[j, t + 8:t + 12] = np.asarray([det.flag[k][row]], "<i4").view(np.uint8)
        out[j, :8] = np.asarray([mask], "<u8").view(np.uint8)
    return out


def model_unpack(det, ids, rec):
    """the rule applied to a copy of det's state: -> snapshot"""
    st = det.snapshot()
    _, slots = model_layout(det.roles, det.windows)
    for j, i in enumerate(ids):
        mask = int(rec[j, :8].view("<u8")[0])
        for k, sl in enumerate(slots):
            if sl is None:
                continue
            row = det.lookup[k][i]
            if row < 0:
                continue
            h, t = sl
            w = det.windows[k]
            hist, seen, flag = st[k]
            if (mask >> k) & 1:
                hist[:w - 1, row] = rec[j, h:h + 4 * (w - 1)].view("<f4")
                seen[row] = rec[j, t:t + 8].view("<i8")[0]
                flag[row] = rec[j, t + 8:t + 12].view("<i4")[0]
            else:
                hist[:w - 1, row] = 0
                seen[row] = 0
                flag[row] = det.cooldowns[k] if det.roles[k] == WAKE else 0
    return st


def same_state(a, b):
    return all(np.array_equal(x.view(np.uint8), y.view(np.uint8)) for p, q in zip(a, b) for x, y in zip(p, q))


# ---- layout -------------------------------------------------------------------------------------------------------------------
def test_layout_sizes_worked_out_by_hand():
    # plain detectors: mask 16; window 5 -> 4 floats = 16; seen, flag, 0 = 16
    assert layout([WAKE], [5]) == (48, [16], [32])
    assert layout([WAKE], [1]) == (32, [16], [16])
    # window 32: 31 floats = 124 -> 128
    assert layout([WAKE], [32]) == (160, [16], [144])
    # WAKE 5, VAD 10 (9 floats = 36 -> 48), OFF: 16 + 32 + 64
    assert layout([WAKE, VAD, OFF], [5, 10, 7]) == (112, [16, 48, -1], [32, 96, -1])
    # OFF first: no bytes for it
    assert layout([OFF, WAKE, WAKE], [3, 2, 3]) == (16 + 32 + 32, [-1, 16, 48], [-1, 32, 64])
    # 64 models of window 1: a 16-byte tail each
    rb, h, t = layout([WAKE] * 64, [1] * 64)
    assert rb == 16 + 64 * 16 and h == t == [16 + 16 * k for k in range(64)]
    for roles, windows in (([WAKE], [5]), ([WAKE, VAD, OFF], [5, 10, 7]), ([OFF, WAKE, VAD, WAKE], [1, 32, 5, 1])):
        rb, slots = model_layout(roles, windows)
        got = layout(roles, windows)
        assert got[0] == rb and rb % 16 == 0
        assert [None if s is None else s for s in slots] == [None if a < 0 else (a, b) for a, b in zip(got[1], got[2])]


def test_header_layout_is_the_one_place_that_knows_the_offsets():
    src = open(os.path.join(CSRC, "mww_detector_records.h")).read()
    assert src.count("detector_record_pad16(") >= 3 and "inline DetRecLayout detector_record_layout(" in src
    for f in ("mww_detector_records.cu", "mww_detector_capi.cu"):
        text = open(os.path.join(CSRC, f)).read()
        assert "pad16" not in text and "hist_off" not in text and "tail_off" not in text, f


# ---- pack and unpack against the model ------------------------------------------------------------------------------------------
CASES = {
    "plain w5": (300, [WAKE], [5], [25], [None]),
    "plain w1": (77, [WAKE], [1], [3], [None]),
    "plain w32": (45, [WAKE], [32], [0], [None]),
    "three models": (120, [WAKE, WAKE, VAD], [5, 32, 1], [10, 0, 7], ["all", "half", "most"]),
    "with OFF": (90, [OFF, VAD, WAKE], [9, 5, 32], [4, 4, 4], [None, "half", "most"]),
}


def _sets(kind, n, rng):
    if kind is None or kind == "all":
        return None
    p = 0.5 if kind == "half" else 0.85
    return np.flatnonzero(rng.random(n) < p).astype(np.int32)


def _case(name, seed, n_ids=None, streams=None):
    n, roles, windows, cooldowns, kinds = CASES[name]
    n = n_ids or n
    rng = np.random.default_rng(seed)
    sets = streams if streams is not None else [_sets(k, n, rng) for k in kinds]
    return Det(n, roles, windows, cooldowns, sets, rng), rng


def _sixty_four(seed, n=50, streams=None):
    rng = np.random.default_rng(seed)
    roles = [WAKE] * 64
    roles[5], roles[17], roles[63] = VAD, OFF, OFF
    windows = [[1, 5, 32][k % 3] for k in range(64)]
    cooldowns = list(rng.integers(0, 30, 64))
    if streams is None:
        streams = [None if k % 4 == 0 else np.flatnonzero(rng.random(n) < 0.6).astype(np.int32) for k in range(64)]
    return Det(n, roles, windows, cooldowns, streams, rng), rng


@pytest.mark.parametrize("name", sorted(CASES) + ["64 models"])
def test_pack_is_the_rule(name):
    det, rng = _sixty_four(1) if name == "64 models" else _case(name, 1)
    ids = np.concatenate([rng.permutation(det.n_ids)[:det.n_ids // 2], [0, det.n_ids - 1, 0]]).astype(np.int32)   # one id twice
    before = det.snapshot()
    got = det.pack(ids)
    assert np.array_equal(got, model_pack(det, ids))
    assert same_state(det.snapshot(), before)                                  # export does not change the detector
    if len(det.roles) == 1:
        assert (got[:, 0] & 1).all()                                           # a plain detector's bit 0 is always set


@pytest.mark.parametrize("name", sorted(CASES) + ["64 models"])
def test_import_into_other_row_counts_and_stream_sets(name):
    """export from one detector, import into one with another id count and other stream sets: members whose bit is set take
    the slot, members whose bit is clear start fresh, non-members ignore the slot, unlisted rows keep every byte"""
    if name == "64 models":
        src, rng = _sixty_four(2)
        dst, _ = _sixty_four(3, n=80)
    else:
        src, rng = _case(name, 2)
        dst, _ = _case(name, 3, n_ids=src.n_ids + 37)
    out_ids = rng.permutation(src.n_ids)[: src.n_ids * 2 // 3].astype(np.int32)
    rec = src.pack(out_ids)
    in_ids = rng.permutation(dst.n_ids)[:out_ids.size].astype(np.int32)
    want = model_unpack(dst, in_ids, rec)
    before = dst.snapshot()
    dst.unpack(in_ids, rec)
    got = dst.snapshot()
    assert same_state(got, want)
    # every kind of slot occurred where the model has a stream set of its own
    taken = fresh = ignored = 0
    for k in range(len(dst.roles)):
        if dst.roles[k] == OFF:
            continue
        mem_dst = dst.lookup[k][in_ids] >= 0
        mem_src = src.lookup[k][out_ids] >= 0
        taken += int((mem_dst & mem_src).sum())
        fresh += int((mem_dst & ~mem_src).sum())
        ignored += int((~mem_dst & mem_src).sum())
        # unlisted rows: every byte as before
        listed = np.zeros(max(dst.streams[k].size, 1), bool)
        listed[dst.lookup[k][in_ids][mem_dst]] = True
        h0, s0, f0 = before[k]
        h1, s1, f1 = got[k]
        assert np.array_equal(h1[:, ~listed].view(np.uint32), h0[:, ~listed].view(np.uint32))
        assert np.array_equal(s1[~listed], s0[~listed]) and np.array_equal(f1[~listed], f0[~listed])
    assert taken > 0
    if any(s is not None and s.size < src.n_ids for s in src.inv):
        assert fresh > 0 and ignored > 0


def test_round_trip_is_bit_exact_and_fresh_rows_are_a_reset():
    det, rng = _case("three models", 4)
    ids = rng.permutation(det.n_ids).astype(np.int32)
    rec = det.pack(ids)
    twin, _ = _case("three models", 5, streams=[None if s.size == det.n_ids else s for s in det.streams])
    twin.unpack(ids, rec)
    used = lambda d: [(h[:w - 1, :s.size], e[:s.size], f[:s.size]) for (h, e, f), s, w in zip(d.snapshot(), d.streams, d.windows)]
    assert same_state(used(twin), used(det))
    # records with every bit clear: every member row of the listed ids gets what a reset gives
    empty = rec.copy()
    empty[:, :8] = 0
    twin.unpack(ids, empty)
    for k, (h, s, f) in enumerate(twin.snapshot()):
        n = twin.streams[k].size
        assert not h[:twin.windows[k] - 1, :n].any() and not s[:n].any()
        assert (f[:n] == (twin.cooldowns[k] if twin.roles[k] == WAKE else 0)).all()


# ---- layout mismatches ------------------------------------------------------------------------------------------------------------
def _layout(multi, roles, windows, cooldowns):
    from microwakeword_b200 import _lib
    L = _lib.MwwDetectorLayout()
    L.multi, L.n_models = multi, len(roles)
    for k, (r, w, c) in enumerate(zip(roles, windows, cooldowns)):
        L.role[k] = r
        L.window[k] = w if r != OFF else 0
        L.cooldown_slices[k] = c if r == WAKE else 0
    L.record_bytes = layout(roles, [w if r != OFF else 1 for r, w in zip(roles, windows)])[0]
    return L


def mismatch(src, dst):
    idx = ctypes.c_int(-2)
    buf = ctypes.create_string_buffer(32)
    if not emul().emul_detrec_mismatch(ctypes.addressof(src), ctypes.addressof(dst), ctypes.byref(idx), buf, 32):
        return None
    return buf.value.decode(), idx.value


def test_each_layout_mismatch_names_its_field():
    base = ([WAKE, WAKE, VAD], [5, 3, 9], [10, 4, 0])
    dst = _layout(1, *base)
    assert mismatch(_layout(1, *base), dst) is None
    # a VAD's cooldown is not compared
    src = _layout(1, *base)
    src.cooldown_slices[2] = 7
    assert mismatch(src, dst) is None
    assert mismatch(_layout(0, *base), dst) == ("multi", -1)
    assert mismatch(_layout(1, [WAKE, WAKE], [5, 3], [10, 4]), dst) == ("n_models", -1)
    assert mismatch(_layout(1, [WAKE, VAD, WAKE], [5, 3, 9], [10, 4, 0]), dst) == ("role", 1)
    assert mismatch(_layout(1, [WAKE, WAKE, VAD], [5, 4, 9], [10, 4, 0]), dst) == ("window", 1)
    assert mismatch(_layout(1, [WAKE, WAKE, VAD], [5, 3, 9], [10, 5, 0]), dst) == ("cooldown_slices", 1)
    src = _layout(1, *base)
    src.record_bytes += 16
    assert mismatch(src, dst) == ("record_bytes", -1)
    # the first field that differs is named
    assert mismatch(_layout(1, [WAKE, WAKE, VAD], [6, 3, 9], [11, 5, 0]), dst) == ("window", 0)
    # an OFF model's window and cooldown are not compared
    off = ([WAKE, OFF], [5, 3], [1, 2])
    src = _layout(0, *off)
    src.window[1], src.cooldown_slices[1] = 9, 9
    assert mismatch(src, _layout(0, *off)) is None
    # plain detectors: window, cooldown
    assert mismatch(_layout(0, [WAKE], [5], [25]), _layout(0, [WAKE], [5], [26])) == ("cooldown_slices", 0)
    assert mismatch(_layout(0, [WAKE], [4], [25]), _layout(0, [WAKE], [5], [25])) == ("window", 0)


# ---- build and ABI ----------------------------------------------------------------------------------------------------------------
NEW = ("mww_get_detector_layout", "mww_export_detector_rows", "mww_import_detector_rows")


def test_new_symbols_are_declared_and_exported_with_their_arguments():
    from microwakeword_b200 import _lib, build
    L = _lib.lib()
    assert all(n in _lib.EXPORTS and hasattr(L, n) for n in NEW)
    syms = subprocess.run(["nm", "-D", "--defined-only", build.OUT], capture_output=True, text=True, check=True).stdout
    assert all(re.search(r"\bT %s\b" % n, syms) for n in NEW)
    hdr = open(os.path.join(ROOT, "include", "mww.h")).read()
    flat = re.sub(r"\s+", " ", re.sub(r"/\*.*?\*/", "", hdr, flags=re.S))
    assert "int mww_get_detector_layout(const mww_detector_t *d, mww_detector_layout *out);" in flat
    assert ("int mww_export_detector_rows(mww_detector_t *d, const int32_t *h_ids, int n, void *d_records, mww_detector_layout *out, "
            "void *cu_stream);") in flat
    assert ("int mww_import_detector_rows(mww_detector_t *d, const int32_t *h_ids, int n, const void *d_records, "
            "const mww_detector_layout *layout, void *cu_stream);") in flat
    body = hdr[hdr.index("typedef struct mww_detector_layout {"):hdr.index("} mww_detector_layout;")]
    assert re.sub(r"\s+", " ", body).endswith("int64_t record_bytes; int32_t multi, n_models; int32_t role[64], window[64], cooldown_slices[64]; ")
    assert [n for n, _ in _lib.MwwDetectorLayout._fields_] == ["record_bytes", "multi", "n_models", "role", "window", "cooldown_slices"]
    assert ctypes.sizeof(_lib.MwwDetectorLayout) == 8 + 8 + 3 * 64 * 4
    vp, i32 = ctypes.c_void_p, ctypes.c_int
    for n in ("mww_export_detector_rows", "mww_import_detector_rows"):
        assert getattr(L, n).argtypes == [vp, vp, i32, vp, ctypes.POINTER(_lib.MwwDetectorLayout), vp]
    # the existing call families keep their names
    assert not any(n.startswith(("mww_detector_", "mww_multi_detector_")) for n in NEW)


def test_null_detector_and_layout_are_refused_without_device_work():
    from microwakeword_b200 import _lib
    L = _lib.lib()
    lay = _lib.MwwDetectorLayout()
    ids = (ctypes.c_int32 * 1)(0)
    assert L.mww_get_detector_layout(None, ctypes.byref(lay)) == -1 and b"detector" in L.mww_last_error(None)
    assert L.mww_export_detector_rows(None, ids, 1, None, None, None) == -1 and b"NULL" in L.mww_last_error(None)
    assert L.mww_import_detector_rows(None, ids, 1, None, ctypes.byref(lay), None) == -1 and b"layout" in L.mww_last_error(None)


def _res_usage(so):
    from microwakeword_b200 import _lib, build
    tool = os.path.join(os.path.dirname(build.NVCC), "cuobjdump")
    if not os.path.exists(tool):
        pytest.skip("cuobjdump is not installed next to nvcc")
    _lib.lib()
    return subprocess.run([tool, "-res-usage", so], capture_output=True, text=True, check=True).stdout


def test_companion_library_holds_exactly_its_two_kernels_without_spills():
    from microwakeword_b200 import build
    assert os.path.basename(build.DR_OUT) == "libmww_detector_records.so" and build.DR_SOURCES == ["mww_detector_records.cu"]
    res = _res_usage(build.DR_OUT)
    found = re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", res)
    names = sorted(n for n, *_ in found)
    assert len(names) == 2 and any("pack_detector_rows_kernel" in n and "unpack" not in n for n in names) \
        and any("unpack_detector_rows_kernel" in n for n in names), res
    assert all(int(stack) == int(local) == 0 for _, _, stack, local in found), found
    flags = [f for f in build.FLAGS if f not in ("-shared", "-cudart", "static")]
    rep = subprocess.run([build.NVCC] + flags + ["-cubin", "-Xptxas", "-v", "-o", os.path.join(_BUILD.name, "detrec.cubin"),
                                                 os.path.join(CSRC, "mww_detector_records.cu")], capture_output=True, text=True, check=True).stderr
    spills = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", rep)
    assert len(spills) == 2 and all(int(a) == int(b) == int(c) == 0 for a, b, c in spills), rep
    # libmww_b200.so holds none of them and finds the library next to itself
    assert "detector_rows_kernel" not in _res_usage(build.OUT)
    if shutil.which("readelf"):
        dyn = subprocess.run(["readelf", "-d", build.OUT], capture_output=True, text=True, check=True).stdout
        assert "[libmww_detector_records.so]" in dyn and "$ORIGIN" in dyn


def test_stale_check_covers_the_companion_library(monkeypatch):
    from microwakeword_b200 import build
    real = os.path.exists
    monkeypatch.setattr(os.path, "exists", lambda p: False if p == build.DR_OUT else real(p))
    assert build._stale()


# ---- Python ------------------------------------------------------------------------------------------------------------------------
def _bare(cls, **attrs):
    """a detector object without a library handle: what the argument checks see before any call"""
    d = object.__new__(cls)
    d.__dict__.update(attrs)
    return d


def test_python_refusals_before_the_library_is_called():
    import torch
    from microwakeword_b200 import _lib
    from microwakeword_b200.detection import DetectorRecords, MultiModelDetector, StreamDetector, _record_ids
    for ids in ([[0, 1]], [0.5], [True, False], np.zeros((2, 2), np.int32), [2 ** 40], torch.zeros(2, dtype=torch.float32)):
        with pytest.raises(ValueError):
            _record_ids(ids, "rows")
    for ids in ([3, 1, 3], np.asarray([2, 0], np.int64), torch.tensor([4, 5], dtype=torch.int32), []):
        got = _record_ids(ids, "rows")
        assert got.dtype == np.int32 and got.flags.c_contiguous and got.tolist() == [int(v) for v in ids]

    class NoLib:
        def __getattr__(self, name):
            raise AssertionError("the library was called: %s" % name)

    lay = _lib.MwwDetectorLayout()
    lay.record_bytes, lay.multi, lay.n_models = 48, 0, 1
    plain = _bare(StreamDetector, _L=NoLib(), device=0, n_rows=8)
    good = torch.zeros((2, 48), dtype=torch.uint8)                         # on the CPU: another device than the detector's
    for data in (good, torch.zeros((2, 48), dtype=torch.int8), torch.zeros((3, 48), dtype=torch.uint8),
                 torch.zeros((2, 32), dtype=torch.uint8), np.zeros((2, 48), np.uint8)):
        with pytest.raises(ValueError):
            plain.import_rows([0, 1], DetectorRecords(data, lay, np.full(2, 0.5)))
    with pytest.raises(ValueError):
        plain.import_rows([[0, 1]], DetectorRecords(good, lay, np.full(2, 0.5)))
    with pytest.raises(ValueError):
        plain.import_rows([0, 1], DetectorRecords(good, lay, np.full(3, 0.5)))          # one cutoff per record
    with pytest.raises(ValueError):
        plain.export_rows([0.5])
    mlay = _lib.MwwDetectorLayout()
    mlay.record_bytes, mlay.multi, mlay.n_models = 80, 1, 2
    multi = _bare(MultiModelDetector, _L=NoLib(), device=0, n_models=2, roles=[WAKE, VAD])
    with pytest.raises(ValueError):
        multi.import_streams([0, 1], DetectorRecords(torch.zeros((2, 80), dtype=torch.uint8), mlay, [np.full(2, 0.5), np.full(2, 0.5)]))
    with pytest.raises(ValueError):
        multi.import_streams([0, 1], DetectorRecords(torch.zeros((2, 80), dtype=torch.uint8), mlay, [np.full(2, 0.5)]))
    with pytest.raises(ValueError):
        multi.export_streams(np.zeros(3, np.float64))


def test_records_save_and_load(tmp_path):
    import torch
    from microwakeword_b200 import _lib
    from microwakeword_b200.detection import DetectorRecords
    rng = np.random.default_rng(0)
    for multi, cut in ((0, rng.random(5)), (1, [rng.random(5), np.full(5, np.nan), rng.random(5)])):
        lay = _layout(multi, [WAKE, OFF, VAD] if multi else [WAKE], [5, 3, 9] if multi else [5], [10, 0, 0] if multi else [10])
        data = torch.from_numpy(rng.integers(0, 256, (5, lay.record_bytes), dtype=np.uint8))
        r = DetectorRecords(data, lay, cut)
        r.save(tmp_path / "rec.npz")
        back = DetectorRecords.load(tmp_path / "rec.npz", "cpu")
        assert torch.equal(back.data, data) and bytes(back.layout) == bytes(lay)
        if multi:
            assert len(back.cutoffs) == 3 and all(np.array_equal(a, b, equal_nan=True) for a, b in zip(back.cutoffs, cut))
        else:
            assert np.array_equal(back.cutoffs, cut)
    assert isinstance(back.layout, _lib.MwwDetectorLayout)


def test_no_cpu_fallback_without_a_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present; the loud-failure path is exercised on GPU-less hosts")
    tool = os.path.join(ROOT, "tools", "detector_records_time.py")
    res = subprocess.run([sys.executable, tool, "--rounds", "1"], capture_output=True, text=True)
    assert res.returncode != 0 and "CUDA" in res.stderr
