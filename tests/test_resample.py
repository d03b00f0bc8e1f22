"""The input-rate resampler (mww_set_input_rate), the parts that need no GPU: the taps mww_resample_taps gives against
scipy's Kaiser design (within 1 LSB), their symmetry, the partial-sum bound and the quantised frequency response; the
kernel's index and phase math (microwakeword_b200/csrc/mww_resample.h, built with g++ in a temporary directory since the
tree may be read-only) under random call splits against the integer upfirdn oracle; the Python call planning; and the
new kernel's registers and spills."""

import ctypes
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest
import scipy.signal

import resample_oracle as ref
from microwakeword_b200 import _lib
from microwakeword_b200.engine import call_plan, samples16

HERE = os.path.dirname(os.path.abspath(__file__))
_BUILD = tempfile.TemporaryDirectory(prefix="mww_resample_test_")
_emul = None


def emul():
    global _emul
    if _emul is None:
        so = os.path.join(_BUILD.name, "libemul_resample.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "emul_resample.cc")], check=True)
        _emul = ctypes.CDLL(so)
        _emul.emul_call.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_longlong, ctypes.c_void_p]
    return _emul


def taps(rate):
    L = _lib.lib()
    n, l, m = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    assert L.mww_resample_taps(rate, None, 0, ctypes.byref(n), ctypes.byref(l), ctypes.byref(m)) == 0
    out = np.zeros(max(n.value, 1), np.int32)
    assert L.mww_resample_taps(rate, out.ctypes.data, out.size, None, None, None) == 0
    return out[:n.value], l.value, m.value


def test_rates_and_refusals():
    L = _lib.lib()
    n, l, m = ctypes.c_int(-1), ctypes.c_int(), ctypes.c_int()
    assert L.mww_resample_taps(16000, None, 0, ctypes.byref(n), ctypes.byref(l), ctypes.byref(m)) == 0
    assert (n.value, l.value, m.value) == (0, 1, 1)
    for bad in (0, -8000, 11025, 16001, 96000):
        assert L.mww_resample_taps(bad, None, 0, None, None, None) == -5      # MWW_EUNSUPPORTED
    want = {8000: (2, 1), 22050: (320, 441), 24000: (2, 3), 32000: (1, 2), 44100: (160, 441), 48000: (1, 3)}
    for rate, lm in want.items():
        assert taps(rate)[1:] == lm


@pytest.mark.parametrize("rate", ref.RATES)
def test_taps_match_kaiser_design(rate):
    h, L, M = taps(rate)
    d = ref.design(rate)
    assert h.size == d.size and h.size % 2 == 1
    want = np.clip(np.round(d * 32768), -32768, 32767)
    assert np.abs(h - want).max() <= 1
    assert np.array_equal(h, h[::-1])                      # symmetric: linear phase
    assert np.abs(h).max() <= 32767
    for p in range(L):                                     # each of the two partial sums of a phase stays inside int32
        ph = np.abs(h[p::L].astype(np.int64))
        assert ph[0::2].sum() < 65536 and ph[1::2].sum() < 65536


@pytest.mark.parametrize("rate", ref.RATES)
def test_taps_frequency_response(rate):
    h, L, M = taps(rate)
    fs_up = rate * L
    lo, hi = (0.45 * rate, 0.55 * rate) if rate == 8000 else (7500.0, 8500.0)
    w, H = scipy.signal.freqz(h / 32768.0 / L, worN=1 << 17, fs=fs_up)
    mag = np.abs(H)
    assert np.abs(mag[w <= lo] - 1).max() <= 4e-4              # passband ripple (the header states 0.0004)
    assert 20 * np.log10(mag[w >= hi].max()) <= -70.0           # stopband


def _emul_stream(rate, x, splits):
    """x int16 [S, N] through the emulated kernel in calls of the given lengths -> the concatenated 16 kHz samples"""
    E = emul()
    h, L, M = taps(rate)
    H = -(-h.size // L)
    S = x.shape[0]
    hist = np.zeros((S, H), np.int16)
    outs, seen = [], 0
    for n in splits:
        chunk = np.ascontiguousarray(x[:, seen:seen + n])
        n_out = samples16(seen, n, rate)
        y = np.zeros((S, max(n_out, 1)), np.int16)
        assert E.emul_call(rate, hist.ctypes.data, chunk.ctypes.data, S, n, seen, y.ctypes.data) == n_out
        outs.append(y[:, :n_out])
        seen += n
    return np.concatenate(outs, 1) if outs else np.zeros((S, 0), np.int16)


@pytest.mark.parametrize("rate", ref.RATES)
@pytest.mark.parametrize("seed", range(3))
def test_emulated_kernel_matches_upfirdn_under_random_splits(rate, seed):
    rng = np.random.default_rng(seed * 1000 + rate)
    h, L, M = taps(rate)
    N = int(rng.integers(1, 3 * rate // 10))
    x = rng.integers(-32768, 32768, (3, N)).astype(np.int16)
    signs = np.where(h[::L][::-1] < 0, -32768, 32767)
    x[0] = np.resize(signs, N)                             # full scale with the signs of one phase's taps: outputs saturate
    x[1] = (rng.standard_normal(N) * 3000).astype(np.int16)
    want = ref.resample(x, h, rate)
    splits, left = [], N
    while left > 0:
        n = int(rng.choice([0, 1, M - 1 if M > 1 else 2, M, M + 1, int(rng.integers(1, 2 * M + 300))]))
        n = min(n, left)
        splits.append(n)
        left -= n
    splits.insert(int(rng.integers(0, len(splits) + 1)), 0)
    got = _emul_stream(rate, x, splits)
    assert got.shape == want.shape
    assert np.array_equal(got, want), (rate, np.flatnonzero((got != want).any(0))[:5])
    assert np.array_equal(_emul_stream(rate, x, [N]), want)


@pytest.mark.parametrize("rate", ref.RATES)
def test_thirty_ms_calls_yield_480_samples(rate):
    if rate * 3 % 100:
        pytest.skip("30 ms is not a whole number of samples at this rate")
    n = rate * 3 // 100
    seen = 0
    for _ in range(50):
        assert samples16(seen, n, rate) == 480
        seen += n
    rows, steps, buffered, pending = call_plan(0, n, 160, [0], [3], rate, 0)
    assert (rows, steps, buffered, pending) == (1, [0], 320, [1])


def test_call_plan_at_16k_unchanged():
    assert call_plan(100, 1000, 160, [1, 0], [3, 2]) == call_plan(100, 1000, 160, [1, 0], [3, 2], 16000, 12345)


def test_resample_kernel_has_no_spills():
    from microwakeword_b200 import build
    cuobjdump = os.path.join(os.path.dirname(build.NVCC), "cuobjdump")
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump is not installed next to nvcc")
    res = subprocess.run([cuobjdump, "-res-usage", build.RS_OUT], capture_output=True, text=True, check=True).stdout
    found = re.findall(r"Function (\S*resample_kernel\S*):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", res)
    assert len(found) == 2, res[-2000:]
    for name, reg, stack, local in found:
        assert int(stack) == 0 and int(local) == 0, name
