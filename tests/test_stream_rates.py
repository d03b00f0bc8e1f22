"""Per-stream input rates (mww_set_stream_rates), the parts that need no GPU: the N identity of include/mww.h for every rate,
mww_rate_inputs against the Python formula, the resampler stage of a per-stream-rate handle emulated on the CPU
(tests/emul_stream_rates.cc: run_rates_tile's planning and resample_kernel's MemberRows body, built with g++ in a temporary
directory since the tree may be read-only) against the integer upfirdn oracle under random rates, splits and rate changes,
the Python planning and refusals, the new symbols, and the kernels: the gathered instantiations do not spill and the
contiguous ones keep the instructions they had before per-stream rates."""

import ctypes
import hashlib
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

import resample_oracle as ref
from microwakeword_b200 import _lib
from microwakeword_b200.engine import (INPUT_RATES, RATE_PER_STREAM, StreamEngine, call_plan, inputs_for_rates, rate_inputs,
                                       resampler_history_len)

HERE = os.path.dirname(os.path.abspath(__file__))
_BUILD = tempfile.TemporaryDirectory(prefix="mww_stream_rates_test_")
_emul = None


def emul():
    global _emul
    if _emul is None:
        so = os.path.join(_BUILD.name, "libemul_stream_rates.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "emul_stream_rates.cc")], check=True)
        _emul = ctypes.CDLL(so)
        vp = ctypes.c_void_p
        _emul.emul_rates_call.argtypes = [vp, ctypes.c_int, vp, ctypes.c_int, vp, ctypes.c_longlong, ctypes.c_longlong, ctypes.c_int,
                                          ctypes.c_int, vp]
        _emul.emul_rate_inputs.restype = ctypes.c_longlong
        _emul.emul_rate_inputs.argtypes = [ctypes.c_int, ctypes.c_longlong]
    return _emul


def ratio(rate):
    return (1, 1) if rate == 16000 else ref.ratio(rate)


def taps(rate):
    L = _lib.lib()
    n = ctypes.c_int()
    assert L.mww_resample_taps(rate, None, 0, ctypes.byref(n), None, None) == 0
    out = np.zeros(max(n.value, 1), np.int32)
    assert L.mww_resample_taps(rate, out.ctypes.data, out.size, None, None, None) == 0
    return out[:n.value]


def oracle(x, rate):
    """int16 [N] at `rate` -> its ceil(N L / M) samples at 16 kHz (the identity at 16 kHz)"""
    return np.asarray(x, np.int16).copy() if rate == 16000 else ref.resample(np.asarray(x, np.int16)[None], taps(rate), rate)[0]


# ---- the N identity ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rate", INPUT_RATES)
def test_n_identity_every_even_t(rate):
    L, M = ratio(rate)
    t = np.arange(0, 1_000_001, 2, dtype=np.int64)
    N = t * M // L
    assert np.array_equal(-(-N * L // M), t)
    if rate == 8000:                                   # odd t is where 8 kHz breaks it: t - 1 samples
        assert np.array_equal(-(-((t + 1) * M // L) * L // M), t)


@pytest.mark.parametrize("rate", INPUT_RATES)
def test_n_identity_random_large_t_and_rate_inputs(rate):
    L, M = ratio(rate)
    lib, E = _lib.lib(), emul()
    rng = np.random.default_rng(rate)
    got = ctypes.c_longlong()
    for t in [0, 2, 2 ** 40] + [2 * int(v) for v in rng.integers(0, 2 ** 39, 300)]:
        N = t * M // L
        assert -(-N * L // M) == t
        assert rate_inputs(t, rate) == N == E.emul_rate_inputs(rate, t)
        assert lib.mww_rate_inputs(rate, t, ctypes.byref(got)) == 0 and got.value == N
    assert lib.mww_rate_inputs(11025, 100, ctypes.byref(got)) == -5
    assert lib.mww_rate_inputs(rate, -2, ctypes.byref(got)) == -1
    assert lib.mww_rate_inputs(rate, 2, None) == -1


def test_thirty_ms_inputs_and_history_lengths():
    want = {8000: 240, 16000: 480, 24000: 720, 32000: 960, 44100: 1323, 48000: 1440}
    for rate, d in want.items():
        assert {int(v) for v in inputs_for_rates([rate] * 3, 480 * np.arange(1, 4).sum(), 480)} == {d}
        assert all(rate_inputs(t + 480, rate) - rate_inputs(t, rate) == d for t in range(0, 480 * 50, 480))
    d22 = [rate_inputs(t + 480, 22050) - rate_inputs(t, 22050) for t in range(0, 480 * 40, 480)]
    assert set(d22) == {661, 662} and sum(d22) == rate_inputs(480 * 40, 22050)
    H = {r: resampler_history_len(r) for r in INPUT_RATES}
    assert H == {8000: 52, 16000: 0, 22050: 111, 24000: 122, 32000: 163, 44100: 222, 48000: 243}
    assert resampler_history_len(RATE_PER_STREAM) == 243 == emul().emul_max_history()


# ---- the resampler stage on the CPU ----------------------------------------------------------------------------------
def _run(rates_per_call, calls, S, tile, seed):
    """Feeds S streams through the emulated stage: calls[i] = n16 of call i, rates_per_call[i] the rates in force.  Returns
    (per-stream 16 kHz output, per-stream oracle output, final history, oracle history)."""
    E = emul()
    rng = np.random.default_rng(seed)
    Hmax = resampler_history_len(RATE_PER_STREAM)
    stride = Hmax + 1
    hist = np.zeros((S, stride), np.int16)
    t = 0
    got = [[] for _ in range(S)]
    # per stream: the inputs since its last rate change, led by N(t_change, r) zeros, and the t of that change
    since, t_change = [[] for _ in range(S)], [0] * S
    prev = list(rates_per_call[0])
    for n16, rates in zip(calls, rates_per_call):
        for s in range(S):
            if rates[s] != prev[s]:                   # a new client at another rate: its history is zeroed
                hist[s] = 0
                since[s], t_change[s] = [np.zeros(rate_inputs(t, rates[s]), np.int16)], t
        prev = list(rates)
        D = inputs_for_rates(rates, t, n16)
        pitch = int(D.max()) + int(rng.integers(0, 3))
        x = np.full((S, max(pitch, 1)), 12345, np.int16)               # padding past D_s must not be read
        for s in range(S):
            x[s, :D[s]] = (rng.standard_normal(D[s]) * 6000).clip(-32768, 32767).astype(np.int16)
            since[s].append(x[s, :D[s]].copy())
        y = np.zeros((S, max(n16, 1)), np.int16)
        r32 = np.ascontiguousarray(rates, np.int32)
        assert E.emul_rates_call(r32.ctypes.data, S, hist.ctypes.data, stride, x.ctypes.data, x.shape[1], t, n16, tile, y.ctypes.data) == 0
        for s in range(S):
            got[s].append(y[s, :n16].copy())
        t += n16
    want, want_hist = [], []
    for s in range(S):
        xin = np.concatenate(since[s]) if since[s] else np.zeros(0, np.int16)
        out = oracle(xin, prev[s])
        assert out.size == t                           # the N identity: exactly t outputs
        want.append(out[t_change[s]:])
        H = resampler_history_len(prev[s])
        want_hist.append(np.concatenate([np.zeros(H, np.int16), xin])[-H:] if H else np.zeros(0, np.int16))
    got_since = [np.concatenate(g)[t_change[s]:] if g else np.zeros(0, np.int16) for s, g in enumerate(got)]
    return got_since, want, hist, want_hist


@pytest.mark.parametrize("seed", range(4))
def test_emulated_stage_random_rates_and_even_splits(seed):
    rng = np.random.default_rng(seed)
    S = 15
    rates = [INPUT_RATES[i] for i in rng.integers(0, len(INPUT_RATES), S)]
    rates[:7] = INPUT_RATES                          # every rate, the identity plan included
    calls = [int(rng.choice([0, 2, 4, 480, 882, 2 * int(rng.integers(1, 2000))])) for _ in range(8)]
    got, want, hist, want_hist = _run([rates] * len(calls), calls, S, int(rng.integers(1, S + 1)), seed)
    for s in range(S):
        assert np.array_equal(got[s], want[s]), (s, rates[s])
        H = resampler_history_len(rates[s])
        assert np.array_equal(hist[s, :H], want_hist[s]), (s, rates[s])


@pytest.mark.parametrize("seed", range(3))
def test_emulated_stage_rate_changes_mid_sequence(seed):
    rng = np.random.default_rng(100 + seed)
    S, n_calls = 9, 10
    rates = [list(INPUT_RATES) + [48000, 8000]]
    for _ in range(n_calls - 1):
        r = list(rates[-1])
        for s in rng.choice(S, int(rng.integers(0, 4)), replace=False):
            r[s] = INPUT_RATES[int(rng.integers(0, len(INPUT_RATES)))]
        rates.append(r)
    calls = [2 * int(rng.integers(0, 1500)) for _ in range(n_calls)]
    got, want, hist, want_hist = _run(rates, calls, S, int(rng.integers(1, 5)), seed)
    for s in range(S):
        assert np.array_equal(got[s], want[s]), s
        H = resampler_history_len(rates[-1][s])
        assert np.array_equal(hist[s, :H], want_hist[s]), s


def test_thirty_ms_live_calls_at_22050_alternate():
    rates = [22050, 16000, 8000, 44100]
    got, want, _, _ = _run([rates] * 12, [480] * 12, 4, 3, 9)
    for s in range(4):
        assert np.array_equal(got[s], want[s])


# ---- Python planning and refusals -------------------------------------------------------------------------------------
def test_call_plan_per_stream_rates():
    # n_samples is n16: the plan equals a 16 kHz plan of the same length
    assert call_plan(100, 960, 160, [1, 0], [3, 2], RATE_PER_STREAM, 4800) == call_plan(100, 960, 160, [1, 0], [3, 2])
    for bad in (1, 481, -2):
        with pytest.raises(ValueError):
            call_plan(0, bad, 160, [0], [3], RATE_PER_STREAM, 0)
    D = inputs_for_rates([8000, 16000, 22050, 48000], 0, 480)
    assert D.dtype == np.int32 and D.tolist() == [240, 480, 661, 1440]
    assert inputs_for_rates([22050], 480, 480).tolist() == [662]


class _FakeEngine(StreamEngine):
    """the argument checks of StreamEngine without a handle: rate, counter and stream rates are given"""

    def __init__(self, rate, t, rates):
        self.n_streams, self._fake = len(rates), (rate, t, np.asarray(rates, np.int32))

    def _rate(self):
        return self._fake[:2]

    @property
    def stream_rates(self):
        return self._fake[2]

    def close(self):
        pass


def test_engine_refusals_before_the_library():
    e = _FakeEngine(RATE_PER_STREAM, 480, [8000, 22050, 48000])
    assert e.inputs_for(480).tolist() == [240, 662, 1440]
    assert e._call_len(1440, 480) == 480 and e._call_len(1500, 0) == 0
    for width, n16 in ((1439, 480), (1440, None), (1440, 479), (1440, -2), (1440, 2.5)):
        with pytest.raises(ValueError):
            e._call_len(width, n16)
    with pytest.raises(ValueError):
        e.inputs_for(3)
    single = _FakeEngine(48000, 0, [48000] * 3)
    assert single._call_len(1440, None) == 1440
    with pytest.raises(ValueError):
        single._call_len(1440, 480)
    with pytest.raises(ValueError):
        single.inputs_for(480)
    import torch
    with pytest.raises(ValueError):                    # float64 (and a host tensor) are refused as on every engine
        e.predict_clip(torch.zeros((3, 1440), dtype=torch.float64), samples16=480)
    with pytest.raises(ValueError):
        e.predict_clip_host(np.zeros((3, 1440), np.float64), samples16=480)
    with pytest.raises(ValueError):
        e.predict_clip_host(np.zeros((3, 1000), np.int16), samples16=480)


def test_engine_without_gpu_fails_loudly():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    with pytest.raises(_lib.MwwError) as e:
        StreamEngine(None, 4, 0, stream_rates=[8000, 16000, 44100, 48000])
    assert e.value.code == -3
    with pytest.raises(ValueError):
        StreamEngine(None, 4, 0, input_rate=48000, stream_rates=[8000] * 4)


# ---- symbols and kernels ----------------------------------------------------------------------------------------------
def test_new_symbols_are_exported():
    from microwakeword_b200 import build
    _lib.lib()
    new = ("mww_set_stream_rates", "mww_get_stream_rates", "mww_rate_inputs")
    assert all(n in _lib.EXPORTS for n in new)
    syms = subprocess.run(["nm", "-D", "--defined-only", build.OUT], capture_output=True, text=True, check=True).stdout
    assert all(re.search(r"\bT %s\b" % n, syms) for n in new)
    header = open(os.path.join(os.path.dirname(HERE), "include", "mww.h")).read()
    assert "#define MWW_RATE_PER_STREAM 0" in header and _lib.MWW_RATE_PER_STREAM == 0


def _cuobjdump():
    from microwakeword_b200 import build
    tool = os.path.join(os.path.dirname(build.NVCC), "cuobjdump")
    if not os.path.exists(tool):
        pytest.skip("cuobjdump is not installed next to nvcc")
    _lib.lib()
    return tool


def test_gathered_resample_kernels_have_no_spills():
    from microwakeword_b200 import build
    res = subprocess.run([_cuobjdump(), "-res-usage", build.RR_OUT], capture_output=True, text=True, check=True).stdout
    found = re.findall(r"Function (\S*resample_kernel\S*):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", res)
    assert len(found) == 2 and all("MemberRows" in name for name, *_ in found), res[-2000:]
    for name, reg, stack, local in found:
        assert int(stack) == 0 and int(local) == 0, name


# sha256 of the instruction encodings (the /* 0x... */ words of cuobjdump -sass, in order) of resample_kernel<int16_t> and
# resample_kernel<float> as built before per-stream rates; the kernel's names now carry the TileRows argument
SASS_BEFORE = {
    "s": "dfabd763910d101a08e1d1178ec8b11e6a473ea0543009ec28e0f7a1bb5a2ac2",
    "f": "f289b613c3db879c9058ae07fab7f7791be130cb375c0acf04fa5eb883dc0886",
}


def test_contiguous_resample_kernels_sass_unchanged():
    from microwakeword_b200 import build
    text = subprocess.run([_cuobjdump(), "-sass", build.RS_OUT], capture_output=True, text=True, check=True).stdout
    words, name = {}, None
    for line in text.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1)
            words[name] = []
        elif name:
            words[name] += re.findall(r"/\* (0x[0-9a-f]{16}) \*/", line)
    got = {}
    for name, w in words.items():
        m = re.match(r"_ZN3mww15resample_kernelI([sf])NS_8TileRowsE", name)
        assert m, name                                 # nothing but the two contiguous instantiations
        got[m.group(1)] = hashlib.sha256(" ".join(w).encode()).hexdigest()
    assert got == SASS_BEFORE
