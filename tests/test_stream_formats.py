"""Per-stream sample formats (mww_set_stream_formats, the _mixed entry points), the parts that need no GPU: the resampler
stage of a handle with per-stream rates and formats emulated on the CPU (tests/emul_stream_formats.cc: run_rates_tile's
planning, MixedRows and the kernel's per-stream format dispatch, built with g++ in a temporary directory since the tree may
be read-only) against "decode with the G.711 / float32 rule, then the integer upfirdn oracle" under random rates, formats,
splits and format changes; the byte-width planning; the Python refusals; the new symbols; and the new library's kernel."""

import ctypes
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

import resample_oracle as ref
from microwakeword_b200 import _lib
from microwakeword_b200.audio.audio_utils import to_int16
from microwakeword_b200.engine import (FORMAT_BYTES, INPUT_RATES, RATE_PER_STREAM, SAMPLE_FORMATS, MultiModelEngine, StreamEngine,
                                       bytes_for_formats, format_codes, inputs_for_rates, rate_inputs, resampler_history_len)
from test_g711 import alaw_ref, ulaw_ref
from test_stream_rates import oracle as resample16

HERE = os.path.dirname(os.path.abspath(__file__))
_BUILD = tempfile.TemporaryDirectory(prefix="mww_stream_formats_test_")
_emul = []
vp, i32, ll = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong
S16, ULAW, ALAW, F32 = (SAMPLE_FORMATS[k] for k in ("s16", "ulaw", "alaw", "f32"))


def emul():
    if not _emul:
        so = os.path.join(_BUILD.name, "libemul_stream_formats.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "emul_stream_formats.cc")], check=True)
        L = ctypes.CDLL(so)
        L.emul_formats_call.argtypes = [vp, vp, i32, vp, i32, vp, ll, ll, i32, i32, vp]
        L.emul_mixed_rows_width.restype = ll
        L.emul_mixed_rows_width.argtypes = [vp, vp, i32, i32, ll, i32]
        _emul.append(L)
    return _emul[0]


def decode(raw: np.ndarray, fmt: int) -> np.ndarray:
    """a stream's samples in format `fmt` (int16, uint8 codes or float32) -> int16, by the rules of include/mww.h"""
    if fmt == ULAW:
        return ulaw_ref(raw)
    if fmt == ALAW:
        return alaw_ref(raw)
    if fmt == F32:
        with np.errstate(invalid="ignore", over="ignore"):
            return np.where(np.isnan(raw), 0, to_int16(np.nan_to_num(raw, nan=0.0))).astype(np.int16)
    return raw.astype(np.int16)


def samples(rng, n, fmt):
    """n random samples of format fmt, as the dtype a row of that format holds"""
    if fmt in (ULAW, ALAW):
        return rng.integers(0, 256, n).astype(np.uint8)
    if fmt == F32:
        x = (rng.standard_normal(n) * 0.4).astype(np.float32)
        x[rng.random(n) < 0.01] = 1.5                  # clamped
        x[rng.random(n) < 0.005] = np.nan              # NaN -> 0
        return x
    return (rng.standard_normal(n) * 8000).clip(-32768, 32767).astype(np.int16)


def mixed_rows(parts, pitch, pad=0xA5):
    """per stream its samples (any dtype) -> uint8 [S, pitch] rows, bytes past each row's own length set to `pad`"""
    x = np.full((len(parts), pitch), pad, np.uint8)
    for s, p in enumerate(parts):
        b = np.ascontiguousarray(p).view(np.uint8)
        x[s, :b.size] = b
    return x


def _run(rates, formats_per_call, calls, tile, seed):
    """Feeds len(rates) streams through the emulated stage; formats_per_call[i] = the formats of call i.  Returns the
    per-stream 16 kHz outputs and histories with their oracles."""
    E = emul()
    rng = np.random.default_rng(seed)
    S = len(rates)
    stride = resampler_history_len(RATE_PER_STREAM) + 1
    hist = np.zeros((S, stride), np.int16)
    r32 = np.ascontiguousarray(rates, np.int32)
    t, got, decoded = 0, [[] for _ in range(S)], [[] for _ in range(S)]
    for n16, fmts in zip(calls, formats_per_call):
        f8 = np.ascontiguousarray(fmts, np.uint8)
        D = inputs_for_rates(rates, t, n16)
        B = bytes_for_formats(rates, fmts, t, n16)
        assert np.array_equal(B, D * FORMAT_BYTES[np.asarray(fmts)])
        parts = [samples(rng, int(D[s]), int(fmts[s])) for s in range(S)]
        pitch = (int(B.max()) + 3) // 4 * 4 + 4 * int(rng.integers(0, 3))
        x = mixed_rows(parts, max(pitch, 4))
        y = np.zeros((S, max(n16, 1)), np.int16)
        assert E.emul_formats_call(r32.ctypes.data, f8.ctypes.data, S, hist.ctypes.data, stride, x.ctypes.data, x.shape[1], t, n16, tile,
                                   y.ctypes.data) == 0
        for s in range(S):
            got[s].append(y[s, :n16].copy())
            decoded[s].append(decode(parts[s], int(fmts[s])))
        t += n16
    for s in range(S):
        xin = np.concatenate(decoded[s]) if decoded[s] else np.zeros(0, np.int16)
        want = resample16(xin, int(rates[s]))
        assert want.size == t
        assert np.array_equal(np.concatenate(got[s]) if got[s] else np.zeros(0, np.int16), want), (s, rates[s])
        H = resampler_history_len(int(rates[s]))
        want_hist = np.concatenate([np.zeros(H, np.int16), xin])[-H:] if H else np.zeros(0, np.int16)
        assert np.array_equal(hist[s, :H], want_hist), (s, rates[s])


# ---- the resampler stage on the CPU ----------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(4))
def test_emulated_stage_random_rates_formats_and_splits(seed):
    rng = np.random.default_rng(seed)
    S = 16
    rates = [INPUT_RATES[i] for i in rng.integers(0, len(INPUT_RATES), S)]
    rates[:7] = INPUT_RATES                          # every rate, the identity plan included
    fmts = [int(f) for f in rng.integers(0, 4, S)]
    fmts[:4] = [S16, ULAW, ALAW, F32]
    calls = [int(rng.choice([0, 2, 4, 480, 882, 2 * int(rng.integers(1, 2000))])) for _ in range(6)]
    _run(rates, [fmts] * len(calls), calls, int(rng.integers(1, S + 1)), seed)


@pytest.mark.parametrize("seed", range(3))
def test_emulated_stage_format_changes_between_calls(seed):
    rng = np.random.default_rng(50 + seed)
    rates = list(INPUT_RATES) + [8000, 8000, 48000]
    S, n_calls = len(rates), 8
    fmts = [[int(f) for f in rng.integers(0, 4, S)]]
    for _ in range(n_calls - 1):
        f = list(fmts[-1])
        for s in rng.choice(S, int(rng.integers(1, 5)), replace=False):
            f[s] = int(rng.integers(0, 4))
        fmts.append(f)
    _run(rates, fmts, [2 * int(rng.integers(0, 1200)) for _ in range(n_calls)], int(rng.integers(1, 5)), seed)


def test_thirty_ms_calls_at_22050_every_format():
    # 661 / 662 samples in turn at 22.05 kHz, one stream per format at each of 22.05, 8 and 48 kHz
    rates = [22050] * 4 + [8000] * 4 + [48000] * 4
    fmts = [S16, ULAW, ALAW, F32] * 3
    _run(rates, [fmts] * 10, [480] * 10, 5, 7)


# ---- byte widths ------------------------------------------------------------------------------------------------------
def test_bytes_per_stream_and_tile_widths():
    E = emul()
    rng = np.random.default_rng(9)
    for _ in range(40):
        S = int(rng.integers(1, 40))
        rates = np.array([INPUT_RATES[i] for i in rng.integers(0, len(INPUT_RATES), S)], np.int32)
        fmts = rng.integers(0, 4, S).astype(np.uint8)
        t, n16 = 2 * int(rng.integers(0, 10 ** 6)), 2 * int(rng.integers(0, 3000))
        B = bytes_for_formats(rates, fmts, t, n16)
        assert np.array_equal(B, inputs_for_rates(rates, t, n16) * np.array([2, 1, 1, 4])[fmts])
        first = int(rng.integers(0, S))
        n = int(rng.integers(1, S - first + 1))
        assert E.emul_mixed_rows_width(rates.ctypes.data, fmts.ctypes.data, first, n, t, n16) == B[first:first + n].max()
    # 30 ms: mu-law at 8 kHz is 240 bytes, int16 at 16 kHz 960, float32 at 48 kHz 5 760, A-law at 22.05 kHz 661 or 662
    assert bytes_for_formats([8000, 16000, 48000, 22050], [ULAW, S16, F32, ALAW], 0, 480).tolist() == [240, 960, 5760, 661]
    assert bytes_for_formats([22050], [ALAW], 480, 480).tolist() == [662]


def test_format_codes():
    assert format_codes(["s16", "ulaw", "alaw", "f32", 0, 3], 6).tolist() == [0, 1, 2, 3, 0, 3]
    assert format_codes("ulaw", 3).tolist() == [1, 1, 1]
    assert SAMPLE_FORMATS["ulaw"] == _lib.MWW_G711_ULAW and SAMPLE_FORMATS["alaw"] == _lib.MWW_G711_ALAW
    for bad in (["pcmu"], [4], [-1], [True], ["S16"], [1.0]):
        with pytest.raises(ValueError):
            format_codes(bad, 1)
    with pytest.raises(ValueError):
        format_codes(["s16", "f32"], 3)


# ---- Python refusals --------------------------------------------------------------------------------------------------
class _FakeEngine(StreamEngine):
    """the argument checks of StreamEngine without a handle: rate, counter, stream rates and formats are given"""

    def __init__(self, rate, t, rates, formats):
        self.n_streams, self._fake = len(rates), (rate, t, np.asarray(rates, np.int32), format_codes(formats, len(rates)))

    def _rate(self):
        return self._fake[:2]

    @property
    def stream_rates(self):
        return self._fake[2]

    @property
    def stream_formats(self):
        return self._fake[3]

    def close(self):
        pass


def test_engine_refusals_before_the_library():
    e = _FakeEngine(RATE_PER_STREAM, 480, [8000, 22050, 48000], ["ulaw", "s16", "f32"])
    assert e.bytes_for(480).tolist() == [240, 1324, 5760]
    assert e._mixed_len(5760, 5760, 1024, 480) == 480 and e._mixed_len(0, 0, 0, 0) == 0
    for width, stride, ptr, n16 in ((5759, 5760, 0, 480), (5760, 5762, 0, 480), (5762, 5762, 0, 480), (5760, 5760, 2, 480),
                                    (5760, 5760, 0, None), (5760, 5760, 0, 479)):
        with pytest.raises(ValueError):
            e._mixed_len(width, stride, ptr, n16)
    rows = np.zeros((3, 5760), np.uint8)
    with pytest.raises(ValueError):                    # law= together with mixed=True
        e.predict_clip_host(rows, samples16=480, law="ulaw", mixed=True)
    for audio in (np.zeros((3, 2880), np.int16), np.zeros((3, 1440), np.float32), np.zeros((3, 5760), np.int8)):
        with pytest.raises(ValueError):                # mixed rows are bytes
            e.predict_clip_host(audio, samples16=480, mixed=True)
    with pytest.raises(ValueError):                    # uint8 without law= or mixed=True is still refused
        e.predict_clip_host(rows, samples16=480)
    with pytest.raises(ValueError):                    # rows too short for the float32 stream
        e.predict_clip_host(np.zeros((3, 5756), np.uint8), samples16=480, mixed=True)
    with pytest.raises(ValueError):                    # a pitch that is not a multiple of 4
        e.predict_clip_host(np.zeros((3, 5762), np.uint8), samples16=480, mixed=True)
    with pytest.raises(ValueError):
        e.predict_clip_remote(0, 5760, samples16=480, mixed=True, law="alaw")
    with pytest.raises(ValueError):
        e.predict_clip_remote(0, 5760, samples16=480, mixed=True, dtype=np.int16)
    single = _FakeEngine(48000, 0, [48000] * 3, "s16")
    with pytest.raises(ValueError):                    # mixed rows need per-stream rates
        single._mixed_len(5760, 5760, 0, 480)
    with pytest.raises(ValueError):
        single.predict_clip_host(rows, samples16=480, mixed=True)


def test_stream_formats_need_stream_rates():
    for cls, first in ((StreamEngine, None), (MultiModelEngine, [None])):
        with pytest.raises(ValueError):
            cls(first, 4, 0, stream_formats=["ulaw"] * 4)


def test_engine_without_gpu_fails_loudly():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    with pytest.raises(_lib.MwwError) as e:
        StreamEngine(None, 4, 0, stream_rates=[8000] * 4, stream_formats="ulaw")
    assert e.value.code == -3


# ---- symbols and kernels ----------------------------------------------------------------------------------------------
NEW = ("mww_set_stream_formats", "mww_get_stream_formats", "mww_features_mixed", "mww_predict_clip_mixed", "mww_predict_clip_multi_mixed",
       "mww_predict_clip_host_mixed", "mww_predict_clip_host_multi_mixed", "mww_predict_clip_remote_mixed",
       "mww_predict_clip_remote_multi_mixed")


def test_new_symbols_are_exported_and_codes_declared():
    from microwakeword_b200 import build
    L = _lib.lib()
    assert all(n in _lib.EXPORTS and hasattr(L, n) for n in NEW)
    syms = subprocess.run(["nm", "-D", "--defined-only", build.OUT], capture_output=True, text=True, check=True).stdout
    assert all(re.search(r"\bT %s\b" % n, syms) for n in NEW)
    header = open(os.path.join(os.path.dirname(HERE), "include", "mww.h")).read()
    for name, code in (("S16", 0), ("ULAW", 1), ("ALAW", 2), ("F32", 3)):
        assert "#define MWW_FORMAT_%s %d" % (name, code) in header and getattr(_lib, "MWW_FORMAT_" + name) == code


def _cuobjdump():
    from microwakeword_b200 import build
    tool = os.path.join(os.path.dirname(build.NVCC), "cuobjdump")
    if not os.path.exists(tool):
        pytest.skip("cuobjdump is not installed next to nvcc")
    _lib.lib()
    return tool


def _res_usage(path):
    res = subprocess.run([_cuobjdump(), "-res-usage", path], capture_output=True, text=True, check=True).stdout
    return {name: tuple(int(v) for v in vals) for name, *vals in
            re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", res)}


def test_mixed_library_holds_exactly_its_kernel():
    from microwakeword_b200 import build
    got = _res_usage(build.RM_OUT)
    assert list(got) == ["_ZN3mww15resample_kernelINS_6Mixed8ENS_9MixedRowsEEEvNS_12ResampleArgsEPKT_PsT0_"], got
    reg, stack, shared, local = next(iter(got.values()))
    assert stack == 0 and local == 0
    # the int16 member kernel's occupancy (256 threads; registers allocated in 8s per thread) and shared memory
    s16 = _res_usage(build.RR_OUT)["_ZN3mww15resample_kernelIsNS_10MemberRowsEEEvNS_12ResampleArgsEPKT_PsT0_"]
    per_sm = lambda r: 65536 // (256 * ((r + 7) // 8 * 8))
    assert per_sm(reg) == per_sm(s16[0]) and shared == s16[2], (reg, s16)
    needed = subprocess.run(["readelf", "-d", build.OUT], capture_output=True, text=True, check=True).stdout
    assert "libmww_resample_mixed.so" in needed
