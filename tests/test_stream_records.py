"""Stream records (mww_export_streams / mww_import_streams), the parts that need no GPU: the record layout against sizes
worked out by hand, the pack and unpack kernels' per-word bodies (microwakeword_b200/csrc/mww_records.h, built with g++ in a
temporary directory) over every rotation of every okay_nabu ring on host buffers, the layout comparison that refuses an
import, the engine's id checks, the instruction SASS of every kernel the library had before stream records, which must not
change, and the register report of the two new kernels."""

import ctypes
import json
import os
import re
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from conftest import GOLDEN
from test_model_streams import sass_functions

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "microwakeword_b200", "csrc")
_BUILD = tempfile.TemporaryDirectory(prefix="mww_records_test_")
_emul = None

HEADER, CARRY, ESTIMATE = 16, 960, 160
FRONTEND = HEADER + CARRY + ESTIMATE                    # 1136
# okay_nabu: first-conv ring 2 x 40, then the rotating rings (rows, channels): blocks 0..3 and the head
RINGS = [(4, 32), (10, 64), (14, 64), (22, 64), (16, 64)]
STATE_ELEMS = 80 + sum(r * c for r, c in RINGS)         # 4176


def emul():
    global _emul
    if _emul is None:
        so = os.path.join(_BUILD.name, "libemul_records.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "emul_records.cc")], check=True)
        _emul = ctypes.CDLL(so)
        _emul.emul_record_model_hash.restype = ctypes.c_uint64
        _emul.emul_record_model_hash.argtypes = [ctypes.c_uint64, ctypes.c_int, ctypes.c_longlong]
    return _emul


def _p(a):
    if a is None:
        return None
    p = ctypes.c_void_p(a.ctypes.data)
    p.array = a                  # a temporary stays alive as long as its pointer
    return p


def _ll(v):
    return np.asarray(v, np.int64)


def layout(state_bytes, pend_bytes):
    K = len(state_bytes)
    out = np.zeros(3 + 2 * K, np.int64)
    emul().emul_record_layout(_p(_ll(state_bytes)), _p(_ll(pend_bytes)), K, _p(out))
    return dict(record_bytes=int(out[0]), carry=int(out[1]), estimate=int(out[2]), nn=out[3:3 + K].tolist(), pend=out[3 + K:].tolist())


def test_assumed_geometry_is_the_kernels():
    src = open(os.path.join(CSRC, "mww_nn_live.cuh")).read()
    assert "kLiveRingRows[5] = {%s}" % ", ".join(str(r) for r, _ in RINGS) in src
    assert "return i == 0 ? 32 : 64;" in src
    assert "kStateFloats = %d" % STATE_ELEMS in open(os.path.join(CSRC, "mww_nn_dev.cuh")).read()


# ---- layout ------------------------------------------------------------------------------------------------------------
def test_layout_sizes_worked_out_by_hand():
    assert layout([], []) == dict(record_bytes=1136, carry=16, estimate=976, nn=[], pend=[])
    # fp32 okay_nabu: 4176 floats = 16704 bytes, 2 pending rows of 40 floats = 320 bytes
    assert layout([16704], [320]) == dict(record_bytes=1136 + 16704 + 320, carry=16, estimate=976, nn=[1136], pend=[17840])
    # int8 okay_nabu: 4176 bytes, 80 bytes
    assert layout([4176], [80]) == dict(record_bytes=5392, carry=16, estimate=976, nn=[1136], pend=[5312])
    # fp32 + int8 + an int8 run-time geometry with 257 channels: 3 rows of 257 bytes = 771 -> 784, 16 pending rows = 640
    L = layout([16704, 4176, 771], [320, 80, 640])
    assert L["nn"] == [1136, 18160, 22416] and L["pend"] == [17840, 22336, 23200] and L["record_bytes"] == 23840
    # a model without ring state and a one-row pending buffer of 40 bytes -> 48
    assert layout([0], [40]) == dict(record_bytes=1136 + 48, carry=16, estimate=976, nn=[1136], pend=[1136])


def test_layout_parts_are_aligned_and_disjoint():
    rng = np.random.default_rng(0)
    for K in (0, 1, 3, 64):
        sb = [int(v) for v in rng.integers(0, 70000, K)]
        pb = [int(v) for v in 40 * rng.integers(1, 64, K) * rng.choice([1, 4], K)]
        L = layout(sb, pb)
        parts = [(0, 8), (L["carry"], CARRY), (L["estimate"], ESTIMATE)]
        for k in range(K):
            parts += [(L["nn"][k], sb[k]), (L["pend"][k], pb[k])]
        end = 0
        for off, size in parts:
            assert off % 16 == 0 and off >= end
            end = off + size
        assert L["record_bytes"] % 16 == 0 and end <= L["record_bytes"] < end + 16
    full = layout([16704] * 64, [320] * 64)
    assert full["record_bytes"] == 1136 + 64 * 17024


# ---- pack / unpack over rotated rings -------------------------------------------------------------------------------------
class HostModel:
    """Streams of one okay_nabu model on the host, rings rotated by `heads` as the live kernels leave them."""

    def __init__(self, S, dtype, heads, seed):
        rng = np.random.default_rng(seed)
        self.S, self.dtype, self.heads, self.es = S, np.dtype(dtype), list(heads), np.dtype(dtype).itemsize
        self.canonical = rng.integers(-100, 100, (S, STATE_ELEMS)).astype(dtype)
        self.pend = rng.integers(-100, 100, (S, 2, 40)).astype(dtype)
        self.physical = self.rotate(self.canonical, +1)

    def rotate(self, state, sign):
        """canonical -> physical (sign +1: logical row r lies at physical row (head + r) % rows) or back (-1)"""
        out, off = state.copy(), 80
        for (rows, cols), h in zip(RINGS, self.heads):
            ring = state[:, off:off + rows * cols].reshape(-1, rows, cols)
            out[:, off:off + rows * cols] = np.roll(ring, sign * h, axis=1).reshape(-1, rows * cols)
            off += rows * cols
        return out

    def job_args(self):
        offs = np.cumsum([80] + [r * c for r, c in RINGS[:-1]]).astype(np.int32) * self.es
        return (5, _p(offs.astype(np.int32)), _p(np.asarray([c * self.es for _, c in RINGS], np.int32)),
                _p(np.asarray([r for r, _ in RINGS], np.int32)), _p(np.asarray(self.heads, np.int32)))


def move(pack, m, rec, ids, inv=None, fresh=None, k=0, n_models=1, zero_fresh=0):
    sb, pb = _ll([STATE_ELEMS * m.es] * n_models), _ll([80 * m.es] * n_models)
    return emul().emul_record_job(int(pack), k, _p(sb), _p(pb), n_models, *m.job_args(), _p(rec), _p(ids), ids.size, _p(m.physical),
                                  _p(m.pend), None, _p(inv), _p(fresh), zero_fresh)


def head_cases():
    """every (ring, source head, destination head); the other rings sit at seeded heads"""
    rng = np.random.default_rng(5)
    for i, (rows, _) in enumerate(RINGS):
        for hs in range(rows):
            for hd in range(rows):
                src = [int(rng.integers(0, r)) for r, _ in RINGS]
                dst = [int(rng.integers(0, r)) for r, _ in RINGS]
                src[i], dst[i] = hs, hd
                yield src, dst


@pytest.mark.parametrize("dtype,word", [(np.float32, 16), (np.int8, 16)])
def test_every_rotation_packs_canonical_and_unpacks_in_place(dtype, word):
    es = np.dtype(dtype).itemsize
    rb = layout([STATE_ELEMS * es], [80 * es])["record_bytes"]
    src_ids, dst_ids = np.asarray([5, 0, 3, 5], np.int32), np.asarray([8, 2, 0, 4], np.int32)
    for case, (hs, hd) in enumerate(head_cases()):
        a, b = HostModel(7, dtype, hs, 2 * case), HostModel(9, dtype, hd, 2 * case + 1)
        rec = np.full((src_ids.size, rb), 0xAB, np.uint8)
        rec[:, :16] = 0
        before = a.physical.copy()
        assert move(True, a, rec, src_ids) == word
        assert np.array_equal(a.physical, before)                                   # export changes nothing
        assert np.array_equal(rec[:, 1136:1136 + STATE_ELEMS * es].view(dtype), a.canonical[src_ids])
        assert np.array_equal(rec[:, 1136 + STATE_ELEMS * es:].view(dtype).reshape(-1, 2, 40), a.pend[src_ids])
        assert (rec[:, :8].view(np.uint64) == 1).all() and (rec[:, 16:1136] == 0xAB).all()          # its own bit, nothing else
        want, want_pend = b.canonical.copy(), b.pend.copy()
        want[dst_ids], want_pend[dst_ids] = a.canonical[src_ids], a.pend[src_ids]
        fresh = np.full(dst_ids.size, 7, np.int32)
        move(False, b, rec, dst_ids, fresh=fresh)
        assert (fresh == -1).all()
        assert np.array_equal(b.rotate(b.physical, -1), want), (hs, hd)             # moved streams arrive, the others stay
        assert np.array_equal(b.pend, want_pend)


def test_frontend_parts_and_padding():
    S, ids = 6, np.asarray([4, 1, 4], np.int32)
    rng = np.random.default_rng(1)
    carry = rng.integers(-30000, 30000, (S, 480)).astype(np.int16)
    est = rng.integers(0, 1 << 32, (S, 40), dtype=np.uint64).astype(np.uint32)
    rec = np.full((ids.size, 1136), 0xCD, np.uint8)
    L = emul()
    args = (_p(_ll([])), _p(_ll([])), 0, 0, None, None, None, None)
    assert L.emul_record_job(1, -1, *args, _p(rec), _p(ids), ids.size, None, _p(carry), _p(est), None, None, 0) == 16
    assert (rec[:, :16] == 0).all()                                               # the mask word and its padding
    assert np.array_equal(rec[:, 16:976].view(np.int16), carry[ids]) and np.array_equal(rec[:, 976:].view(np.uint32), est[ids])
    carry2, est2 = np.zeros_like(carry), np.zeros_like(est)
    to = np.asarray([0, 5, 2], np.int32)
    L.emul_record_job(0, -1, *args, _p(rec), _p(to), to.size, None, _p(carry2), _p(est2), None, None, 0)
    want_c, want_e = np.zeros_like(carry), np.zeros_like(est)
    want_c[to], want_e[to] = carry[ids], est[ids]
    assert np.array_equal(carry2, want_c) and np.array_equal(est2, want_e)


def test_membership_rule():
    """model 1 of two: a non-member exports a zero slot and a clear bit; on import a non-member destination ignores the
    slot, a member takes a set bit's state, and a member given a clear bit is reported for a fresh start"""
    dtype, es = np.int8, 1
    rb = layout([STATE_ELEMS] * 2, [80] * 2)["record_bytes"]
    a, b = HostModel(3, dtype, [1, 2, 3, 4, 5], 0), HostModel(2, dtype, [3, 9, 0, 21, 15], 1)
    inv_a = np.asarray([0, -1, 1, 2, -1], np.int32)                  # global streams 0, 2, 3 are members of the source model
    src_ids = np.asarray([1, 3, 0, 4], np.int32)
    rec = np.full((4, rb), 0xEE, np.uint8)
    rec[:, :16] = 0
    move(True, a, rec, src_ids, inv=inv_a, k=1, n_models=2)
    slot = slice(1136 + 4176 + 80, 1136 + 4176 + 80 + 4176)
    assert rec[:, :8].view(np.uint64).ravel().tolist() == [0, 2, 2, 0]
    assert (rec[[0, 3], slot.start:] == 0).all() and (rec[:, 1136:slot.start] == 0xEE).all()       # model 0's slot is not this job's
    assert np.array_equal(rec[1, slot].view(np.int8), a.canonical[2]) and np.array_equal(rec[2, slot].view(np.int8), a.canonical[0])
    inv_b = np.asarray([-1, 1, -1, 0], np.int32)                     # destination members: global streams 3, 1
    dst_ids = np.asarray([3, 0, 1, 2], np.int32)                     # bit clear -> member, set -> non-member, set -> member, clear -> non-member
    want = b.canonical.copy()
    want[1] = a.canonical[0]
    fresh = np.full(4, 9, np.int32)
    move(False, b, rec, dst_ids, inv=inv_b, fresh=fresh, k=1, n_models=2)
    assert fresh.tolist() == [0, -1, -1, -1]
    assert np.array_equal(b.rotate(b.physical, -1), want)
    # a model whose fresh state is zeros (fp32, hybrid) gets it from the unpack itself, pending rows included
    want[0], want_pend = 0, b.pend.copy()
    want_pend[0] = 0
    move(False, b, rec, dst_ids, inv=inv_b, k=1, n_models=2, zero_fresh=1)
    assert np.array_equal(b.rotate(b.physical, -1), want) and np.array_equal(b.pend, want_pend)


def test_run_time_geometry_span_is_copied_by_the_widest_word_that_fits():
    L = emul()
    for sb, pb, word in ((771, 640, 1), (772, 640, 4), (776, 640, 8), (784, 640, 16), (0, 40, 8)):
        S = 5
        rng = np.random.default_rng(sb)
        state = rng.integers(0, 255, (S, max(sb, 1)), dtype=np.uint8)[:, :sb].copy()
        pend = rng.integers(0, 255, (S, pb), dtype=np.uint8)
        rb = layout([sb], [pb])["record_bytes"]
        ids = np.asarray([4, 0], np.int32)
        rec = np.full((2, rb), 0x77, np.uint8)
        rec[:, :16] = 0
        args = (_p(_ll([sb])), _p(_ll([pb])), 1, 0, None, None, None, None)
        assert L.emul_record_job(1, 0, *args, _p(rec), _p(ids), 2, _p(state), _p(pend), None, None, None, 0) == word
        pad = (sb + 15) // 16 * 16
        assert np.array_equal(rec[:, 1136:1136 + sb], state[ids]) and (rec[:, 1136 + sb:1136 + pad] == 0).all()
        assert np.array_equal(rec[:, 1136 + pad:1136 + pad + pb], pend[ids]) and (rec[:, 1136 + pad + pb:] == 0).all()
        state2, pend2, fresh = np.zeros_like(state), np.zeros_like(pend), np.zeros(2, np.int32)
        L.emul_record_job(0, 0, *args, _p(rec), _p(ids), 2, _p(state2), _p(pend2), None, None, _p(fresh), 0)
        assert np.array_equal(state2[ids], state[ids]) and np.array_equal(pend2[ids], pend[ids]) and not state2[1:4].any()


# ---- the refusals that are host code -------------------------------------------------------------------------------------
def _layout_struct(**kw):
    from microwakeword_b200 import _lib
    s = _lib.MwwStreamLayout()
    s.record_bytes, s.n_models, s.frontend_buffered, s.hop_samples = 23840, 3, 320, 160
    for k in range(3):
        s.pending_rows[k], s.model_hash[k], s.rows_are_features[k] = k, 1000 + k, 1
    for name, v in kw.items():
        if isinstance(v, tuple):
            getattr(s, name)[v[0]] = v[1]
        else:
            setattr(s, name, v)
    return s


def test_layout_struct_matches_the_header():
    from microwakeword_b200 import _lib
    assert ctypes.sizeof(_lib.MwwStreamLayout) == emul().emul_sizeof_stream_layout() == 856


def test_layout_comparison_names_the_first_field_that_differs():
    L = emul()
    cases = [({}, "", -1), (dict(rows_are_features=(1, 0)), "", -1), (dict(n_models=2), "n_models", -1),
             (dict(model_hash=(2, 7)), "model_hash", 2), (dict(record_bytes=23856), "record_bytes", -1),
             (dict(hop_samples=320), "hop_samples", -1), (dict(frontend_buffered=0), "frontend_buffered", -1),
             (dict(pending_rows=(1, 0)), "pending_rows", 1),
             (dict(pending_rows=(0, 1), hop_samples=320, model_hash=(1, 5)), "model_hash", 1)]
    for change, field, index in cases:
        buf = ctypes.create_string_buffer(64)
        src, dst = _layout_struct(**change), _layout_struct()
        assert L.emul_layout_mismatch(ctypes.byref(src), ctypes.byref(dst), buf) == index and buf.value.decode() == field, change
    # precision and state size are part of a model's identity
    h = L.emul_record_model_hash
    assert len({h(5, 0, 4176), h(5, 1, 4176), h(5, 0, 4177), h(6, 0, 4176)}) == 4


def test_engine_refuses_bad_id_lists_before_the_library():
    import torch
    from microwakeword_b200.engine import _Engine
    for ids in ([[0, 1]], [0.5], np.zeros((2, 2), np.int32), torch.zeros(2, dtype=torch.float32)):
        with pytest.raises(ValueError):
            _Engine._ids(ids)
    for ids in ([3, 1, 3], np.asarray([2, 0], np.int64), torch.tensor([4, 5], dtype=torch.int32), []):
        got = _Engine._ids(ids)
        assert got.dtype == np.int32 and got.flags.c_contiguous and got.tolist() == [int(v) for v in ids]


def test_no_cpu_fallback_without_a_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present; the loud-failure path is exercised on GPU-less hosts")
    tool = os.path.join(os.path.dirname(HERE), "tools", "stream_records_time.py")
    res = subprocess.run([sys.executable, tool, "--streams", "64"], capture_output=True, text=True)
    assert res.returncode != 0 and "CUDA" in res.stderr


# ---- the kernels that existed before stream records compile to the same instructions; the new ones do not spill ----------
SASS_GOLDEN = os.path.join(GOLDEN, "sass_kernels_before_stream_records.json")


def test_existing_kernels_sass_unchanged():
    from microwakeword_b200 import _lib, build
    _lib.lib()                                               # builds the library if needed
    if not os.path.exists(os.path.join(os.path.dirname(build.NVCC), "cuobjdump")):
        pytest.skip("cuobjdump is not installed next to nvcc")
    got = sass_functions(build.OUT)
    want = json.load(open(SASS_GOLDEN))
    assert len(want) >= 39
    changed = sorted(k for k in want if got.get(k) != want[k])
    assert not changed, changed
    new = sorted(k for k in got if k not in want)
    assert len(new) == 8 and all("pack_streams_kernel" in k for k in new), new          # 2 kernels x 4 word sizes, nothing else


def test_record_kernels_do_not_spill():
    from microwakeword_b200 import build
    if not os.path.exists(build.NVCC):
        pytest.skip("nvcc is not installed")
    flags = [f for f in build.FLAGS if f not in ("-shared", "-cudart", "static")]
    res = subprocess.run([build.NVCC] + flags + ["-cubin", "-Xptxas", "-v", "-o", os.path.join(_BUILD.name, "records.cubin"),
                                                  os.path.join(CSRC, "mww_records.cu")], capture_output=True, text=True, check=True)
    reports = re.findall(r"Function properties for (\S+)\s+(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", res.stderr)
    assert len(reports) == 8 and all("pack_streams_kernel" in name for name, *_ in reports), res.stderr
    assert all(int(stack) == int(st) == int(ld) == 0 for _, stack, st, ld in reports), reports
