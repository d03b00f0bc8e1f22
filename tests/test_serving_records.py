"""Moving a stream's serving state between handles (mww_write_audio_history; mww_export_endpointer_rows /
mww_import_endpointer_rows; StreamRecords.history, Endpointer.export_streams / import_streams), the parts that need no GPU:
the history write body (microwakeword_b200/csrc/mww_history.h, built with g++ in a temporary directory by
tests/emul_serving_records.cc) against NumPy for many row lengths, capacities and counters, in its vector and scalar forms,
followed by the existing read and append bodies (tests/emul_history.cc); the endpointer record layout against sizes worked
out by hand; pack and unpack (mww_serving_records.h) against a NumPy model of the rule in include/mww.h, into endpointers
with other row counts, stream sets and baselines; each layout mismatch and its field; the symbols and their argument lists;
the Python refusals, which happen before the library is called; save / load; the companion library's link, kernels and
registers; the timing tool's loud failure without a GPU."""

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
_BUILD = tempfile.TemporaryDirectory(prefix="mww_serving_records_test_")
_emul = {}


def emul(name="serving_records"):
    if name not in _emul:
        so = os.path.join(_BUILD.name, "libemul_%s.so" % name)
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "emul_%s.cc" % name)], check=True)
        L = ctypes.CDLL(so)
        vp, i32, ll = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong
        if name == "serving_records":
            L.emul_history_write.restype = i32
            L.emul_history_write.argtypes = [vp, i32, ll, vp, i32, i32, vp, ll, i32]
            L.emul_eprec_layout.restype = None
            L.emul_eprec_layout.argtypes = [i32, vp]
            for fn in (L.emul_eprec_pack, L.emul_eprec_unpack):
                fn.restype = None
                fn.argtypes = [vp, ll, vp, vp, i32, vp]
            L.emul_eprec_mismatch.restype = i32
            L.emul_eprec_mismatch.argtypes = [vp, vp, ctypes.c_char_p, i32]
        else:
            L.emul_history_append.restype = i32
            L.emul_history_append.argtypes = [i32, vp, i32, i32, ll, vp, ll, i32, i32]
            L.emul_history_read.restype = i32
            L.emul_history_read.argtypes = [vp, i32, i32, ll, vp, i32, i32, vp, ll]
        _emul[name] = L
    return _emul[name]


def _i32(v):
    return np.ascontiguousarray(v, np.int32)


# ---- the history write ------------------------------------------------------------------------------------------------------------
def write(ring, C, seen, ids, rows, allow_vec=True):
    ids, rows = _i32(ids), np.ascontiguousarray(rows, np.int16)
    n, m = rows.shape
    stride = max(m, 1)
    buf = np.zeros((max(n, 1), stride), np.int16)
    buf[:n, :m] = rows
    return emul().emul_history_write(ring.ctypes.data, C, seen, ids.ctypes.data, n, m, buf.ctypes.data, stride, int(allow_vec))


def model_write(ring, C, seen, ids, rows):
    """the rule: zeros then the row, sample t at position seen - m + t, slot pos mod C"""
    m = rows.shape[1]
    for i, s in enumerate(ids):
        ring[s] = 0
        for t in range(max(0, m - C), m):
            ring[s, (seen - m + t) % C] = rows[i, t]


def model_read(ring, C, seen, s, n):
    pos = np.arange(seen - n, seen)
    return ring[s, pos % C]


@pytest.mark.parametrize("C", [8, 480, 32000])
def test_history_write_is_the_rule(C):
    rng = np.random.default_rng(C)
    S = 6
    for seen in (0, 5, C - 3, 3 * C + 16, 7 * C + 8 * 11, 10 * C + 5):
        for m in sorted({0, 1, 7, 8, C - 1, C, C + 1, 2 * C + 9, 3 * C}):
            ring = rng.integers(-30000, 30000, (S, C)).astype(np.int16)
            ids = [4, 1, 3]
            rows = rng.integers(-30000, 30000, (len(ids), m)).astype(np.int16)
            want = ring.copy()
            model_write(want, C, seen, ids, rows)
            got = ring.copy()
            vec = write(got, C, seen, ids, rows)
            assert np.array_equal(got, want), (seen, m)
            assert vec == (seen % 8 == 0 and m % 8 == 0 and max(m, 1) % 8 == 0)
            scalar = ring.copy()
            assert write(scalar, C, seen, ids, rows, allow_vec=False) == 0
            assert np.array_equal(scalar, got)                   # the vector and scalar forms agree
            assert np.array_equal(got[[0, 2, 5]], ring[[0, 2, 5]])  # other streams keep every byte


def test_read_after_write_gives_the_row_and_appends_continue_it():
    """the existing read body returns the row zero-padded on the left; the existing append body continues it"""
    rng = np.random.default_rng(7)
    h = emul("history")
    for C, seen, m, calls in ((480, 960, 100, [480, 37, 480]), (32000, 16000 * 7 + 5, 40000, [480] * 3), (8, 3, 5, [3, 8]),
                              (32000, 480 * 9, 4801, [480, 480, 1237])):
        S = 3
        ring = rng.integers(-30000, 30000, (S, C)).astype(np.int16)
        rows = rng.integers(-30000, 30000, (S, m)).astype(np.int16)
        write(ring, C, seen, [0, 1, 2], rows)
        stream = [np.concatenate([np.zeros(max(C - m, 0), np.int16), rows[s, -min(m, C):]]) for s in range(S)]
        ids = _i32([2, 0, 1])
        for n in (0, 1, min(m, C), C):
            out = np.zeros((3, max(n, 1)), np.int16)
            h.emul_history_read(ring.ctypes.data, C, S, seen, ids.ctypes.data, 3, n, out.ctypes.data, max(n, 1))
            for i, s in enumerate(ids):
                assert np.array_equal(out[i, :n], stream[s][C - n:]), (C, m, n)
        for n16 in calls:
            audio = rng.integers(-30000, 30000, (S, n16)).astype(np.int16)
            h.emul_history_append(0, ring.ctypes.data, S, C, seen, audio.ctypes.data, n16, n16, 1)
            seen += n16
            stream = [np.concatenate([stream[s], audio[s]]) for s in range(S)]
            for s in range(S):
                assert np.array_equal(model_read(ring, C, seen, s, C), stream[s][-C:])


def test_write_body_lives_beside_the_existing_bodies():
    src = open(os.path.join(CSRC, "mww_history.h")).read()
    for fn in ("history_write_plan(", "history_write_vec_shape(", "history_write_one("):
        assert "MWW_HD" in src[src.rindex("\n", 0, src.index(fn)):src.index(fn)], fn
    cu = open(os.path.join(CSRC, "mww_serving_records.cu")).read()
    assert "history_write_one(" in cu and "history_write_plan(" in cu


# ---- endpointer records: layout ----------------------------------------------------------------------------------------------------
def layout(w):
    out = np.zeros(6, np.int64)
    emul().emul_eprec_layout(w, out.ctypes.data)
    return out.tolist()


def test_layout_sizes_worked_out_by_hand():
    # head 16, segmenter 16, seen + flags 16, two ages 16, then hist[w - 1] padded to 16
    assert layout(5) == [80, 0, 16, 32, 48, 64]
    assert layout(1) == [64, 0, 16, 32, 48, 64]
    assert layout(32) == [64 + 128, 0, 16, 32, 48, 64]            # 31 floats = 124 bytes -> 128
    assert layout(2) == [80, 0, 16, 32, 48, 64] and layout(6) == [96, 0, 16, 32, 48, 64]
    hdr = open(os.path.join(ROOT, "include", "mww.h")).read()
    assert "A\n *     rule of vad_window 5 has 80-byte records" in hdr or "vad_window 5 has 80-byte records" in re.sub(r"\s*\*\s*", " ", hdr)


def test_header_layout_is_the_one_place_that_knows_the_offsets():
    src = open(os.path.join(CSRC, "mww_serving_records.h")).read()
    assert "inline EpRecLayout endpoint_record_layout(" in src
    for f in ("mww_serving_records.cu", "mww_endpoint_capi.cu"):
        text = open(os.path.join(CSRC, f)).read()
        assert "pad16" not in text and not re.search(r"\b(64|80)\b.*record", text), f


# ---- endpointer records: pack and unpack against the model --------------------------------------------------------------------------
class Ep:
    """host state of an endpointer as the kernels see it, with arbitrary bytes everywhere"""

    F = ("seen", "flags", "armed", "elapsed", "run", "silence", "heard", "start", "speech_end")

    def __init__(self, n_streams, members, w, rng, armed_frac=0.5):
        self.n_streams, self.w = n_streams, w
        self.members = _i32(members)
        R = self.members.size
        self.row_of = np.full(n_streams, -1, np.int32)
        self.row_of[self.members] = np.arange(R)
        self.hist = rng.standard_normal((max(w - 1, 1), max(R, 1))).astype(np.float32)
        self.s = {
            "seen": rng.integers(0, 1 << 40, R).astype(np.int64),
            "flags": rng.integers(0, 1 << 63, R, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, R, dtype=np.uint64),
            "armed": np.where(rng.random(R) < armed_frac, self.members, -1).astype(np.int32),
            "elapsed": rng.integers(1, 300, R).astype(np.int32), "run": rng.integers(0, 10, R).astype(np.int32),
            "silence": rng.integers(0, 30, R).astype(np.int32), "heard": rng.integers(0, 2, R).astype(np.int32),
            "start": rng.integers(-(1 << 33), 1 << 33, R).astype(np.int64), "speech_end": rng.integers(-(1 << 33), 1 << 33, R).astype(np.int64),
        }

    def args(self):
        cfg = _i32([self.w, self.members.size, self.n_streams])
        ptrs = (ctypes.c_void_p * 11)(*([self.hist.ctypes.data] + [self.s[k].ctypes.data for k in self.F] + [self.row_of.ctypes.data]))
        return cfg, ptrs

    def pack(self, ids, base):
        ids = _i32(ids)
        rb = layout(self.w)[0]
        rec = np.full((ids.size, rb // 4), 0xA5A5A5A5, np.uint32)
        cfg, p = self.args()
        emul().emul_eprec_pack(cfg.ctypes.data, base, p, ids.ctypes.data, ids.size, rec.ctypes.data)
        return rec.view(np.uint8).reshape(ids.size, rb)

    def unpack(self, ids, base, rec):
        ids, rec = _i32(ids), np.ascontiguousarray(rec)
        cfg, p = self.args()
        emul().emul_eprec_unpack(cfg.ctypes.data, base, p, ids.ctypes.data, ids.size, rec.ctypes.data)

    def snapshot(self):
        return self.hist.copy(), {k: v.copy() for k, v in self.s.items()}


def model_pack(ep, ids, base):
    rb = layout(ep.w)[0]
    out = np.zeros((len(ids), rb), np.uint8)
    for j, i in enumerate(ids):
        r = ep.row_of[i]
        if r < 0:
            continue
        s = ep.s
        armed = s["armed"][r] >= 0
        out[j, 0:8] = np.asarray([1, int(armed)], "<i4").view(np.uint8)
        if armed:
            out[j, 16:32] = np.asarray([s[k][r] for k in ("elapsed", "run", "silence", "heard")], "<i4").view(np.uint8)
            out[j, 48:64] = np.asarray([base - s["start"][r], base - s["speech_end"][r]], "<i8").view(np.uint8)
        out[j, 32:40] = np.asarray([s["seen"][r]], "<i8").view(np.uint8)
        out[j, 40:48] = np.asarray([s["flags"][r]], "<u8").view(np.uint8)
        out[j, 64:64 + 4 * (ep.w - 1)] = ep.hist[:ep.w - 1, r].astype("<f4").view(np.uint8)
    return out


def model_unpack(ep, ids, base, rec):
    hist, s = ep.snapshot()
    for j, i in enumerate(ids):
        r = ep.row_of[i]
        if r < 0:
            continue
        member, armed = rec[j, 0:8].view("<i4")
        if not member:
            hist[:, r] = 0 if ep.w > 1 else hist[:, r]
            for k in ("seen", "flags", "elapsed", "run", "silence", "heard", "start", "speech_end"):
                s[k][r] = 0
            s["armed"][r] = -1
            continue
        s["seen"][r] = rec[j, 32:40].view("<i8")[0]
        s["flags"][r] = rec[j, 40:48].view("<u8")[0]
        if ep.w > 1:
            hist[:ep.w - 1, r] = rec[j, 64:64 + 4 * (ep.w - 1)].view("<f4")
        if armed:
            s["armed"][r] = i
            for q, k in enumerate(("elapsed", "run", "silence", "heard")):
                s[k][r] = rec[j, 16 + 4 * q:20 + 4 * q].view("<i4")[0]
            a0, a1 = rec[j, 48:64].view("<i8")
            s["start"][r], s["speech_end"][r] = base - a0, base - a1
        else:
            s["armed"][r] = -1
            for k in ("elapsed", "run", "silence", "heard", "start", "speech_end"):
                s[k][r] = 0
    return hist, s


def same(a, b):
    return np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32)) and all(np.array_equal(a[1][k], b[1][k]) for k in a[1])


@pytest.mark.parametrize("w", [1, 5, 32])
def test_pack_is_the_rule_and_changes_nothing(w):
    rng = np.random.default_rng(w)
    ep = Ep(300, np.flatnonzero(rng.random(300) < 0.7), w, rng)
    ids = np.concatenate([rng.permutation(300)[:200], [0, 299, 0]]).astype(np.int32)   # non-members, and one id twice
    before = ep.snapshot()
    base = 123456789
    got = ep.pack(ids, base)
    assert np.array_equal(got, model_pack(ep, ids, base))
    assert same(ep.snapshot(), before)
    member = ep.row_of[ids] >= 0
    assert not got[~member].any()                                          # a non-member exports a zero record
    unarmed = member & (ep.s["armed"][np.maximum(ep.row_of[ids], 0)] < 0)
    assert unarmed.any() and not got[unarmed][:, 16:32].any() and not got[unarmed][:, 48:64].any()


@pytest.mark.parametrize("w", [1, 5, 32])
def test_import_into_another_row_count_stream_set_and_baseline(w):
    """armed rows are renumbered and rebased; members take, members of member-0 records reset, non-members ignore; unlisted
    rows keep every byte"""
    rng = np.random.default_rng(10 + w)
    src = Ep(300, np.flatnonzero(rng.random(300) < 0.6), w, rng)
    dst = Ep(437, np.flatnonzero(rng.random(437) < 0.6), w, rng)
    base_src, base_dst = 16000 * 60 + 320, 16000 * 3 + 160          # the destination's axis is younger: positions go negative
    out_ids = rng.permutation(300)[:250].astype(np.int32)
    rec = src.pack(out_ids, base_src)
    in_ids = rng.permutation(437)[:250].astype(np.int32)
    want = model_unpack(dst, in_ids, base_dst, rec)
    before = dst.snapshot()
    dst.unpack(in_ids, base_dst, rec)
    got = dst.snapshot()
    assert same(got, want)
    # each kind occurred
    m_src, m_dst = src.row_of[out_ids] >= 0, dst.row_of[in_ids] >= 0
    armed_src = m_src & (src.s["armed"][np.maximum(src.row_of[out_ids], 0)] >= 0)
    assert (m_dst & armed_src).any() and (m_dst & m_src & ~armed_src).any() and (m_dst & ~m_src).any() and (~m_dst & m_src).any()
    # renumbered and rebased: a taken armed row holds its new id and positions shifted by base_dst - base_src
    for j in np.flatnonzero(m_dst & armed_src):
        r, q = dst.row_of[in_ids[j]], src.row_of[out_ids[j]]
        assert got[1]["armed"][r] == in_ids[j]
        assert got[1]["start"][r] - src.s["start"][q] == base_dst - base_src
        assert got[1]["speech_end"][r] - src.s["speech_end"][q] == base_dst - base_src
    # unlisted rows: every byte as before
    listed = np.zeros(dst.members.size, bool)
    listed[dst.row_of[in_ids][m_dst]] = True
    assert np.array_equal(got[0][:, ~listed].view(np.uint32), before[0][:, ~listed].view(np.uint32))
    assert all(np.array_equal(got[1][k][~listed], before[1][k][~listed]) for k in got[1])


def test_round_trip_is_bit_exact_on_one_axis():
    rng = np.random.default_rng(3)
    a = Ep(200, np.arange(200), 5, rng)
    b = Ep(200, np.arange(200), 5, rng)
    ids = rng.permutation(200).astype(np.int32)
    b.unpack(ids, 777, a.pack(ids, 777))
    ha, sa = a.snapshot()
    hb, sb = b.snapshot()
    assert np.array_equal(ha.view(np.uint32), hb.view(np.uint32))
    armed = sa["armed"] >= 0
    for k in sa:
        if k in ("elapsed", "run", "silence", "heard", "start", "speech_end"):
            assert np.array_equal(sa[k][armed], sb[k][armed]) and not sb[k][~armed].any(), k
        else:
            assert np.array_equal(sa[k], sb[k]), k


# ---- layout mismatches and the time axis ----------------------------------------------------------------------------------------------
def _lay(**kw):
    from microwakeword_b200 import _lib
    L = _lib.MwwEndpointerLayout()
    d = dict(record_bytes=80, vad_window=5, stride=3, hop_samples=160, buffered=320, pending=1, samples_seen=48000, steps=90)
    d.update(kw)
    for k, v in d.items():
        setattr(L, k, v)
    return L


def mismatch(src, dst):
    buf = ctypes.create_string_buffer(32)
    return buf.value.decode() if emul().emul_eprec_mismatch(ctypes.addressof(src), ctypes.addressof(dst), buf, 32) else None


def test_each_layout_mismatch_names_its_field():
    dst = _lay()
    assert mismatch(_lay(), dst) is None
    assert mismatch(_lay(samples_seen=5, steps=0), dst) is None           # the baseline is for information
    for field, v in (("vad_window", 4), ("stride", 2), ("hop_samples", 320), ("buffered", 400), ("pending", 0), ("record_bytes", 96)):
        assert mismatch(_lay(**{field: v}), dst) == field
    assert mismatch(_lay(stride=1, pending=0), dst) == "stride"             # the first field that differs
    src = open(os.path.join(CSRC, "mww_endpoint_capi.cu")).read()
    assert "update the endpointer after the handle's last call" in src and "the records' \" + field + \" differs" in src


# ---- build and ABI ------------------------------------------------------------------------------------------------------------------------
NEW = ("mww_write_audio_history", "mww_get_endpointer_layout", "mww_export_endpointer_rows", "mww_import_endpointer_rows")


def test_new_symbols_are_declared_and_exported_with_their_arguments():
    from microwakeword_b200 import _lib, build
    L = _lib.lib()
    assert all(n in _lib.EXPORTS and hasattr(L, n) for n in NEW)
    syms = subprocess.run(["nm", "-D", "--defined-only", build.OUT], capture_output=True, text=True, check=True).stdout
    assert all(re.search(r"\bT %s\b" % n, syms) for n in NEW)
    hdr = open(os.path.join(ROOT, "include", "mww.h")).read()
    flat = re.sub(r"\s+", " ", re.sub(r"/\*.*?\*/", "", hdr, flags=re.S))
    assert ("int mww_write_audio_history(mww_t *h, const int32_t *h_ids, int n, int n_samples, const int16_t *d_in, long long in_stride, "
            "void *cu_stream);") in flat
    assert "int mww_get_endpointer_layout(const mww_endpointer_t *ep, mww_endpointer_layout *out);" in flat
    assert ("int mww_export_endpointer_rows(mww_endpointer_t *ep, const int32_t *h_ids, int n, void *d_records, mww_endpointer_layout *out, "
            "void *cu_stream);") in flat
    assert ("int mww_import_endpointer_rows(mww_endpointer_t *ep, const int32_t *h_ids, int n, const void *d_records, "
            "const mww_endpointer_layout *layout, void *cu_stream);") in flat
    body = hdr[hdr.index("typedef struct mww_endpointer_layout {"):hdr.index("} mww_endpointer_layout;")]
    body = re.sub(r"\s+", " ", re.sub(r"/\*.*?\*/", "", body))
    assert body.endswith("int64_t record_bytes; int32_t vad_window, stride, hop_samples, buffered, pending, pad; int64_t samples_seen, steps; ")
    assert [n for n, _ in _lib.MwwEndpointerLayout._fields_] == ["record_bytes", "vad_window", "stride", "hop_samples", "buffered",
                                                                "pending", "pad", "samples_seen", "steps"]
    assert ctypes.sizeof(_lib.MwwEndpointerLayout) == 8 + 6 * 4 + 2 * 8
    vp, i32, ll = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong
    assert L.mww_write_audio_history.argtypes == [vp, vp, i32, i32, vp, ll, vp]
    for n in ("mww_export_endpointer_rows", "mww_import_endpointer_rows"):
        assert getattr(L, n).argtypes == [vp, vp, i32, vp, ctypes.POINTER(_lib.MwwEndpointerLayout), vp]
    # the mww_endpointer_* family keeps its call set
    assert not any(n.startswith("mww_endpointer_") for n in NEW)


def test_null_objects_are_refused_without_device_work():
    from microwakeword_b200 import _lib
    L = _lib.lib()
    lay = _lib.MwwEndpointerLayout()
    ids = (ctypes.c_int32 * 1)(0)
    assert L.mww_write_audio_history(None, ids, 1, 8, None, 8, None) == -1
    assert L.mww_get_endpointer_layout(None, ctypes.byref(lay)) == -1 and b"endpointer" in L.mww_last_error(None)
    assert L.mww_export_endpointer_rows(None, ids, 1, None, None, None) == -1 and b"NULL" in L.mww_last_error(None)
    assert L.mww_import_endpointer_rows(None, ids, 1, None, ctypes.byref(lay), None) == -1


def _res_usage(so):
    from microwakeword_b200 import _lib, build
    tool = os.path.join(os.path.dirname(build.NVCC), "cuobjdump")
    if not os.path.exists(tool):
        pytest.skip("cuobjdump is not installed next to nvcc")
    _lib.lib()
    return subprocess.run([tool, "-res-usage", so], capture_output=True, text=True, check=True).stdout


def test_companion_library_holds_exactly_its_three_kernels_without_spills():
    from microwakeword_b200 import build
    assert os.path.basename(build.SR_OUT) == "libmww_serving_records.so" and build.SR_SOURCES == ["mww_serving_records.cu"]
    res = _res_usage(build.SR_OUT)
    found = re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", res)
    names = sorted(n for n, *_ in found)
    assert len(names) == 3, res
    for k in ("history_write_kernel", "pack_endpointer_rows_kernel", "unpack_endpointer_rows_kernel"):
        assert sum(k in n and not (k.startswith("pack") and "unpack" in n) for n in names) == 1, (k, names)
    assert all(int(stack) == int(local) == 0 for _, _, stack, local in found), found
    flags = [f for f in build.FLAGS if f not in ("-shared", "-cudart", "static")]
    rep = subprocess.run([build.NVCC] + flags + ["-cubin", "-Xptxas", "-v", "-o", os.path.join(_BUILD.name, "sr.cubin"),
                                                 os.path.join(CSRC, "mww_serving_records.cu")], capture_output=True, text=True, check=True).stderr
    spills = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", rep)
    assert len(spills) == 3 and all(int(a) == int(b) == int(c) == 0 for a, b, c in spills), rep
    # no other library holds them, and libmww_b200.so finds this one next to itself
    for other in (build.OUT, build.HIST_OUT, build.EP_OUT):
        text = _res_usage(other)
        assert "history_write_kernel" not in text and "endpointer_rows_kernel" not in text, other
    if shutil.which("readelf"):
        dyn = subprocess.run(["readelf", "-d", build.OUT], capture_output=True, text=True, check=True).stdout
        assert "[libmww_serving_records.so]" in dyn and "$ORIGIN" in dyn


def test_stale_check_covers_the_companion_library(monkeypatch):
    from microwakeword_b200 import build
    real = os.path.exists
    monkeypatch.setattr(os.path, "exists", lambda p: False if p == build.SR_OUT else real(p))
    assert build._stale()


# ---- Python ---------------------------------------------------------------------------------------------------------------------------------
class NoLib:
    def __getattr__(self, name):
        raise AssertionError("the library was called: %s" % name)


def _bare(cls, **attrs):
    o = object.__new__(cls)
    o.__dict__.update(attrs)
    return o


def test_endpointer_refusals_before_the_library_is_called():
    import torch
    from microwakeword_b200 import _lib
    from microwakeword_b200.endpoint import Endpointer, EndpointerRecords

    class Eng:
        n_streams = 10

    ep = _bare(Endpointer, _L=NoLib(), device=0, engine=Eng(), n_rows=10)
    for ids in ([[0, 1]], [0.5], [True], [10], [-1], np.zeros((2, 2), np.int32), torch.zeros(2, dtype=torch.float32)):
        with pytest.raises(ValueError):
            ep.export_streams(ids)
    lay = _lib.MwwEndpointerLayout()
    lay.record_bytes = 80
    good = torch.zeros((2, 80), dtype=torch.uint8)                        # on the CPU: another device than the endpointer's
    for data in (good, torch.zeros((2, 80), dtype=torch.int8), torch.zeros((3, 80), dtype=torch.uint8),
                 torch.zeros((2, 64), dtype=torch.uint8), np.zeros((2, 80), np.uint8)):
        with pytest.raises(ValueError):
            ep.import_streams([0, 1], EndpointerRecords(data, lay))
    for ids in ([0, 0], [0, 11], [[0, 1]]):
        with pytest.raises(ValueError):
            ep.import_streams(ids, EndpointerRecords(good, lay))
    with pytest.raises(ValueError):
        ep.import_streams([0, 1], EndpointerRecords(good, _lib.MwwStreamLayout()))


def test_engine_history_refusals_before_the_library_is_called():
    import torch
    from microwakeword_b200 import _lib
    from microwakeword_b200.engine import StreamEngine, StreamRecords
    eng = _bare(StreamEngine, _L=NoLib(), device=0, _h=None)
    eng._dev = lambda: torch.device("cpu")                                 # let the records pass, so the history is checked
    lay = _lib.MwwStreamLayout()
    lay.record_bytes = 32
    data = torch.zeros((2, 32), dtype=torch.uint8)
    for hist in (torch.zeros((2, 8), dtype=torch.int32), torch.zeros((3, 8), dtype=torch.int16), torch.zeros(8, dtype=torch.int16),
                 np.zeros((2, 8), np.int16), torch.zeros((2, (1 << 22) + 8), dtype=torch.int16)):
        with pytest.raises(ValueError):
            eng.import_streams([0, 1], StreamRecords(data, lay, hist))
    for h in (-1, 0.5, True):
        with pytest.raises(ValueError):
            eng.export_streams([0, 1], history=h)


def test_records_save_and_load(tmp_path):
    import torch
    from microwakeword_b200 import _lib
    from microwakeword_b200.endpoint import EndpointerRecords
    from microwakeword_b200.engine import StreamRecords
    rng = np.random.default_rng(0)
    lay = _lay()
    data = torch.from_numpy(rng.integers(0, 256, (5, 80), dtype=np.uint8))
    EndpointerRecords(data, lay).save(tmp_path / "ep.npz")
    back = EndpointerRecords.load(tmp_path / "ep.npz", "cpu")
    assert torch.equal(back.data, data) and bytes(back.layout) == bytes(lay) and isinstance(back.layout, _lib.MwwEndpointerLayout)
    slay = _lib.MwwStreamLayout()
    slay.record_bytes, slay.n_models = 64, 1
    for hist in (None, torch.from_numpy(rng.integers(-30000, 30000, (5, 4801)).astype(np.int16))):
        StreamRecords(data, slay, hist).save(tmp_path / "s.npz")
        back = StreamRecords.load(tmp_path / "s.npz", "cpu")
        assert torch.equal(back.data, data) and bytes(back.layout) == bytes(slay)
        assert (back.history is None) if hist is None else torch.equal(back.history, hist)


def test_docs_say_how_to_bound_the_history_buffer():
    from microwakeword_b200.engine import _Engine
    for text in (_Engine.export_streams.__doc__, open(os.path.join(ROOT, "README.md")).read()):
        assert "batches of ids" in re.sub(r"\s+", " ", text)


def test_no_cpu_fallback_without_a_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present; the loud-failure path is exercised on GPU-less hosts")
    tool = os.path.join(ROOT, "tools", "serving_records_time.py")
    res = subprocess.run([sys.executable, tool, "--rounds", "1"], capture_output=True, text=True)
    assert res.returncode != 0 and "CUDA" in res.stderr
