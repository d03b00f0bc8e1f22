"""Resampled stream records (mww_export_resampled_streams / mww_import_resampled_streams), the parts that need no GPU: the
continuation condition against the integer upfirdn oracle, the 30 ms cadence table, the record layout worked out by hand,
the resampler part through the record emulation (tests/emul_records.cc, built with g++ in a temporary directory) into
handles with other history strides, the symbols and argument types, the engine's refusals and the save / load round trip."""

import ctypes
import os
import re
import subprocess
import tempfile
from math import gcd

import numpy as np
import pytest
import torch

import resample_oracle as ref
from conftest import ROOT
from microwakeword_b200 import _lib
from microwakeword_b200.engine import INPUT_RATES, RATE_PER_STREAM, StreamEngine, StreamRecords, rate_inputs, resampler_history_len

HERE = os.path.dirname(os.path.abspath(__file__))
_BUILD = tempfile.TemporaryDirectory(prefix="mww_resampled_records_test_")
_emul = None

PART = 496                                       # int16 hist[244], padded to 16
H = {8000: 52, 16000: 0, 22050: 111, 24000: 122, 32000: 163, 44100: 222, 48000: 243}
STRIDE = {r: (h + 1) // 2 * 2 for r, h in H.items()}
STRIDE[RATE_PER_STREAM] = 244


def emul():
    global _emul
    if _emul is None:
        so = os.path.join(_BUILD.name, "libemul_resampled_records.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "emul_resampled_records.cc")], check=True)
        _emul = ctypes.CDLL(so)
        vp = ctypes.c_void_p
        _emul.emul_resampler_job_shape.argtypes = [ctypes.c_longlong, ctypes.c_int, vp]
        _emul.emul_resampler_job.argtypes = [ctypes.c_int, ctypes.c_longlong, ctypes.c_int, vp, ctypes.c_longlong, vp, ctypes.c_int, vp]
        _emul.emul_record_layout.argtypes = [vp, vp, ctypes.c_int, vp]
        _emul.emul_resampler_layout_offsets.argtypes = [vp]
    return _emul


def ratio(rate):
    g = gcd(16000, rate)
    return 16000 // g, rate // g


def taps(rate):
    n = ctypes.c_int()
    assert _lib.lib().mww_resample_taps(rate, None, 0, ctypes.byref(n), None, None) == 0
    out = np.zeros(n.value, np.int32)
    assert _lib.lib().mww_resample_taps(rate, out.ctypes.data, out.size, None, None, None) == 0
    return out


# ---- the continuation condition --------------------------------------------------------------------------------------
@pytest.mark.parametrize("rate", ref.RATES)
def test_phase_rule_against_upfirdn(rate):
    """A stream given N inputs continues in a handle that has given it N' inputs, with its last H inputs as history, bit for
    bit exactly when N' = N (mod M), and at another N' some later sample differs."""
    L, M = ratio(rate)
    h, Hr = taps(rate), H[rate]
    assert Hr == -(-h.size // L) == resampler_history_len(rate)
    rng = np.random.default_rng(rate)
    K = 3 * M + 40                                       # later inputs: every phase of the filter is reached
    same = differ = 0
    for trial in range(8):
        N = int(rng.integers(Hr, Hr + 5 * M))
        if trial % 2 == 0:
            Np = N + M * int(rng.integers(-((N - Hr) // M), 4))       # the same phase
        else:
            Np = int(rng.integers(Hr, Hr + 5 * M))
            if M > 1 and Np % M == N % M:
                Np += 1
        x = rng.integers(-20000, 20000, N + K).astype(np.int16)
        want = ref.resample(x[None], h, rate)[0][-(-N * L // M):]
        # the destination: whatever it was given before, then the source's last H inputs as history, then the same later input
        z = np.concatenate([rng.integers(-20000, 20000, Np - Hr).astype(np.int16), x[N - Hr:]])
        got = ref.resample(z[None], h, rate)[0][-(-Np * L // M):]
        n = min(want.size, got.size)
        assert n >= K * L // M - 1
        if Np % M == N % M:
            assert np.array_equal(got[:n], want[:n]), (rate, N, Np)
            same += 1
        else:
            assert not np.array_equal(got[:n], want[:n]), (rate, N, Np)
            differ += 1
    assert (same, differ) == ((4, 4) if M > 1 else (8, 0))


@pytest.mark.parametrize("rate", INPUT_RATES)
def test_per_stream_phase_is_t_mod_L(rate):
    """with per-stream rates N(t, r) mod M is fixed by t mod L (even t), and fixes it where M > 1"""
    L, M = ratio(rate)
    rng = np.random.default_rng(7)
    for t in (2 * rng.integers(0, 1 << 40, 200)).tolist():
        for u in (t + 2 * L * int(rng.integers(-5, 6)), t + 2 * int(rng.integers(1, 4 * L))):
            if u < 0:
                continue
            same_phase = rate_inputs(t, rate) % M == rate_inputs(u, rate) % M
            assert same_phase == (M == 1 or (t - u) % L == 0), (rate, t, u)


def test_thirty_ms_cadence_only_22050_can_mismatch():
    """after c calls of 480 16 kHz samples the phase N(480 c) mod M takes one value at every rate but 22.05 kHz, where it
    follows the parity of c"""
    table = {}
    for rate in INPUT_RATES:
        L, M = ratio(rate)
        table[rate] = sorted({rate_inputs(480 * c, rate) % M for c in range(2000)})
        assert (480 % L == 0) == (rate != 22050)
    assert table == {8000: [0], 16000: [0], 22050: [0, 220], 24000: [0], 32000: [0], 44100: [0], 48000: [0]}
    assert [rate_inputs(480 * c, 22050) % 441 for c in range(4)] == [0, 220, 0, 220]
    assert [480 * c % 320 for c in range(4)] == [0, 160, 0, 160]


# ---- layout --------------------------------------------------------------------------------------------------------------
def _base_layout(state_bytes, pend_bytes):
    out = np.zeros(3 + 2 * len(state_bytes), np.int64)
    sb, pb = np.asarray(state_bytes, np.int64), np.asarray(pend_bytes, np.int64)
    emul().emul_record_layout(sb.ctypes.data, pb.ctypes.data, len(state_bytes), out.ctypes.data)
    return int(out[0])


def _shape(rec_off, stride):
    out = np.zeros(6, np.int64)
    emul().emul_resampler_job_shape(rec_off, stride, out.ctypes.data)
    return dict(zip(("parts", "bytes", "padded", "rec_off", "word", "words"), out.tolist()))


def test_layout_worked_out_by_hand_at_every_rate():
    assert emul().emul_resampler_part_samples() == 244 == max(STRIDE.values())
    assert resampler_history_len(RATE_PER_STREAM) == 243
    # the stream record is unchanged; the part follows it: frontend only, int8 okay_nabu, fp32 okay_nabu, both
    for base, models in ((1136, ([], [])), (5392, ([4176], [80])), (18160, ([16704], [320])), (22416, ([16704, 4176], [320, 80]))):
        assert _base_layout(*models) == base
        record_bytes, resampler_off = base + PART, base
        assert record_bytes % 16 == 0
        # bytes of the history row, and the widest word dividing it (16 for the empty 16 kHz part)
        want = {8000: (104, 8), 16000: (0, 16), 22050: (224, 16), 24000: (244, 4), 32000: (328, 8), 44100: (444, 4),
                48000: (488, 8), RATE_PER_STREAM: (488, 8)}
        for rate, (nbytes, word) in want.items():
            assert STRIDE[rate] * 2 == nbytes
            assert _shape(resampler_off, STRIDE[rate]) == dict(parts=1, bytes=nbytes, padded=PART, rec_off=resampler_off, word=word,
                                                              words=PART // word), rate


def test_layout_struct_matches_the_header():
    out = np.zeros(7, np.int64)
    emul().emul_resampler_layout_offsets(out.ctypes.data)
    S = _lib.MwwResamplerLayout
    assert out[0] == ctypes.sizeof(S) == 40
    assert out[1:].tolist() == [getattr(S, f).offset for f, _ in S._fields_]


# ---- pack / unpack of the resampler part --------------------------------------------------------------------------------
def _history(S, rate, rng):
    """a history [S][stride] whose first H samples of each row are the stream's, zeros after (every rate in per-stream mode)"""
    if rate == RATE_PER_STREAM:
        rates = [INPUT_RATES[i] for i in rng.integers(0, len(INPUT_RATES), S)]
    else:
        rates = [rate] * S
    hist = np.zeros((S, STRIDE[rate]), np.int16)
    for s, r in enumerate(rates):
        hist[s, :H[r]] = rng.integers(-32768, 32767, H[r])
    return hist, rates


def _pack(hist, stride, ids, base):
    rec_bytes = base + PART
    rec = np.full((ids.size, rec_bytes), 0xAB, np.uint8)       # garbage: every byte of the part is written
    emul().emul_resampler_job(1, base, stride, rec.ctypes.data, rec_bytes, ids.ctypes.data, ids.size, hist.ctypes.data if hist.size else None)
    return rec


def _unpack(rec, hist, stride, ids, base):
    emul().emul_resampler_job(0, base, stride, rec.ctypes.data, rec.shape[1], ids.ctypes.data, ids.size, hist.ctypes.data if hist.size else None)


@pytest.mark.parametrize("src", list(H) + [RATE_PER_STREAM])
def test_pack_writes_the_row_then_zeros(src):
    rng = np.random.default_rng(src)
    S, base = 37, 1136
    hist, _ = _history(S, src, rng)
    ids = rng.permutation(S)[:20].astype(np.int32)
    ids[3] = ids[4]                                             # export allows an id twice
    rec = _pack(hist, STRIDE[src], ids, base)
    assert np.all(rec[:, :base] == 0xAB)                        # the rest of the record is another job's
    part = rec[:, base:].copy().view(np.int16)
    assert part.shape == (ids.size, 248)
    for j, s in enumerate(ids):
        assert np.array_equal(part[j, :STRIDE[src]], hist[s]) and not part[j, STRIDE[src]:].any()


# every move between strides the rule allows: the same rate in either mode; 16 kHz into a per-stream slot at 16000
MOVES = [(r, r) for r in H] + [(r, RATE_PER_STREAM) for r in H] + [(RATE_PER_STREAM, r) for r in H] + [(RATE_PER_STREAM, RATE_PER_STREAM)]


@pytest.mark.parametrize("src,dst", MOVES)
def test_unpack_into_other_strides(src, dst):
    rng = np.random.default_rng(1000 + src + 7 * dst)
    S, D, base = 29, 45, 5392
    # the source's streams all at the destination's rate when it has one, else at the source's
    rate = dst if dst != RATE_PER_STREAM else (src if src != RATE_PER_STREAM else None)
    if rate is None:
        hist, rates = _history(S, RATE_PER_STREAM, rng)
    else:
        hist = np.zeros((S, STRIDE[src]), np.int16)
        hist[:, :H[rate]] = rng.integers(-32768, 32767, (S, H[rate]))
        rates = [rate] * S
    ids = rng.permutation(S)[:17].astype(np.int32)
    rec = _pack(hist, STRIDE[src], ids, base)
    garbage = rng.integers(-32768, 32767, (D, STRIDE[dst])).astype(np.int16)
    dest = garbage.copy()
    dst_ids = rng.permutation(D)[:ids.size].astype(np.int32)
    _unpack(rec, dest, STRIDE[dst], dst_ids, base)
    for j, (s, d) in enumerate(zip(ids, dst_ids)):
        Hr = H[rates[s]]
        assert np.array_equal(dest[d, :Hr], hist[s, :Hr])
        # the destination row's tail comes out zero: the record's zeros past the source row, and past H within it
        assert not dest[d, Hr:].any()
    others = np.setdiff1d(np.arange(D), dst_ids)
    assert np.array_equal(dest[others], garbage[others])


def test_a_row_that_went_from_48_to_8_khz_keeps_a_zero_tail():
    """per-stream mode: set_stream_rates zeroes the whole row and the resampler writes only the first H, so a stream that
    was at 48 kHz and is now at 8 kHz exports 52 samples and zeros, and lands in a single-rate 8 kHz row and back intact"""
    rng = np.random.default_rng(48)
    row = np.zeros((4, 244), np.int16)
    row[2, :243] = rng.integers(-32768, 32767, 243)          # at 48 kHz
    row[2] = 0                                                # mww_set_stream_rates(2 -> 8000) zeroes the stride
    row[2, :52] = rng.integers(-32768, 32767, 52)             # the 8 kHz resampler writes hist[0, 52)
    ids = np.asarray([2], np.int32)
    rec = _pack(row, 244, ids, 1136)
    single = rng.integers(-32768, 32767, (3, 52)).astype(np.int16)
    _unpack(rec, single, 52, np.asarray([1], np.int32), 1136)
    assert np.array_equal(single[1], row[2, :52])
    back = _pack(single, 52, np.asarray([1], np.int32), 1136)
    assert np.array_equal(back, rec)


# ---- the C-ABI and the engine ---------------------------------------------------------------------------------------------
def test_symbols_and_argtypes():
    L = _lib.lib()
    hdr = open(os.path.join(ROOT, "include", "mww.h")).read()
    for name in ("mww_get_resampler_layout", "mww_export_resampled_streams", "mww_import_resampled_streams"):
        assert name in _lib.EXPORTS and hasattr(L, name)
        decl = re.search(r"int %s\((.*?)\);" % name, hdr, re.S).group(1)
        assert len(getattr(L, name).argtypes) == decl.count(",") + 1, name
        assert getattr(L, name).restype is ctypes.c_int32
    P = ctypes.POINTER
    assert L.mww_export_resampled_streams.argtypes[4:6] == [P(_lib.MwwStreamLayout), P(_lib.MwwResamplerLayout)]
    assert L.mww_import_resampled_streams.argtypes[4:6] == [P(_lib.MwwStreamLayout), P(_lib.MwwResamplerLayout)]


def _records(n, base=1136, rate=8000):
    layout = _lib.MwwStreamLayout(record_bytes=base, n_models=0, frontend_buffered=320, hop_samples=160)
    rs = _lib.MwwResamplerLayout(record_bytes=base + PART, resampler_off=base, rate=rate, inputs_seen=4800, samples16_seen=9600)
    data = torch.arange(n * (base + PART), dtype=torch.int64).to(torch.uint8).reshape(n, base + PART)
    return StreamRecords(data, layout, None, rs, np.full(n, rate, np.int32))


class _NoLibrary:
    def __getattr__(self, name):
        raise AssertionError("the library was called: %s" % name)


def _engine():
    e = object.__new__(StreamEngine)
    e._h, e._L, e.device = None, _NoLibrary(), 0
    return e


def test_engine_refuses_malformed_resampled_records_before_the_library():
    e = _engine()
    recs = _records(3)
    for bad in (np.full(2, 8000, np.int32), np.full(3, 8000, np.int64), [8000] * 3, None, np.full((3, 1), 8000, np.int32)):
        r = _records(3)
        r.rates = bad
        with pytest.raises(ValueError, match="rates"):
            e.import_streams([0, 1, 2], r)
    # data sized for the stream record alone, not resampler.record_bytes
    short = StreamRecords(recs.data[:, :1136].contiguous(), recs.layout, None, recs.resampler, recs.rates)
    with pytest.raises(ValueError, match="record_bytes=%d" % (1136 + PART)):
        e.import_streams([0, 1, 2], short)
    with pytest.raises(ValueError, match="history"):
        e.export_streams([0], history=-1, resampler=True)


def test_save_load_round_trip(tmp_path):
    recs = _records(5, base=5392, rate=RATE_PER_STREAM)
    recs.rates = np.asarray([8000, 16000, 22050, 44100, 48000], np.int32)
    recs.history = torch.arange(5 * 7, dtype=torch.int16).reshape(5, 7)
    path = os.path.join(tmp_path, "r.npz")
    recs.save(path)
    got = StreamRecords.load(path, "cpu")
    assert torch.equal(got.data, recs.data) and torch.equal(got.history, recs.history)
    assert got.rates.dtype == np.int32 and np.array_equal(got.rates, recs.rates)
    for f, _ in _lib.MwwResamplerLayout._fields_:
        assert getattr(got.resampler, f) == getattr(recs.resampler, f), f
    assert bytes(got.layout) == bytes(recs.layout)
    # records without a resampler part round-trip without one
    plain = StreamRecords(recs.data[:, :5392].contiguous(), recs.layout)
    plain.save(path)
    got = StreamRecords.load(path, "cpu")
    assert got.resampler is None and got.rates is None and got.history is None


def test_an_old_file_without_the_new_fields_still_loads(tmp_path):
    """a checkpoint written before records carried the resampler: the stream layout's fields, data and audio history"""
    path = os.path.join(tmp_path, "old.npz")
    layout = _lib.MwwStreamLayout(record_bytes=1136, n_models=0, frontend_buffered=320, hop_samples=160)
    fields = {k: np.asarray(getattr(layout, k)) for k in StreamRecords._SCALARS}
    fields.update({k: np.ctypeslib.as_array(getattr(layout, k)).copy() for k in StreamRecords._ARRAYS})
    np.savez(path, data=np.zeros((2, 1136), np.uint8), audio_history=np.ones((2, 4), np.int16), **fields)
    got = StreamRecords.load(path, "cpu")
    assert got.resampler is None and got.rates is None and got.layout.record_bytes == 1136 and got.history.shape == (2, 4)


def test_timing_tool_fails_loudly_without_a_gpu():
    if torch.cuda.is_available():
        pytest.skip("a GPU is present; the loud-failure path is exercised on GPU-less hosts")
    import sys
    tool = os.path.join(ROOT, "tools", "resampled_records_time.py")
    res = subprocess.run([sys.executable, tool, "--streams", "64"], capture_output=True, text=True)
    assert res.returncode != 0 and "CUDA" in res.stderr
