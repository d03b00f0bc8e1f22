"""TEST INFRASTRUCTURE: the integer definition of the input-rate resampler (include/mww.h, mww_set_input_rate), restated
with scipy: upfirdn of the Q15 taps over the zero-stuffed input, the rounding shift and int16 saturation.  float64 is exact
here (every product is below 2^30 and every sum below 2^53).  The product never imports this module."""

from math import ceil, gcd

import numpy as np
import scipy.signal

RATES = (8000, 22050, 24000, 32000, 44100, 48000)


def ratio(rate: int):
    g = gcd(16000, rate)
    return 16000 // g, rate // g


def design(rate: int) -> np.ndarray:
    """the float design the library quantises: scipy's Kaiser method, length made odd, times L"""
    L, _ = ratio(rate)
    fs_up = rate * L
    lo, hi = (0.45 * rate, 0.55 * rate) if rate == 8000 else (7500.0, 8500.0)
    n, beta = scipy.signal.kaiserord(80.0, (hi - lo) / (fs_up / 2))
    return scipy.signal.firwin(n | 1, (lo + hi) / 2, window=("kaiser", beta), fs=fs_up) * L


def resample(x: np.ndarray, taps: np.ndarray, rate: int) -> np.ndarray:
    """int16 [..., N] at `rate` -> the ceil(N L / M) int16 samples at 16 kHz the definition gives"""
    L, M = ratio(rate)
    x = np.asarray(x)
    n_out = -(-x.shape[-1] * L // M)
    flat = x.reshape(-1, x.shape[-1]).astype(np.float64)
    out = np.empty((flat.shape[0], n_out), np.int16)
    h = np.asarray(taps, np.float64)
    for i, row in enumerate(flat):
        y = scipy.signal.upfirdn(h, row, L, M)[:n_out] if row.size else np.zeros(0)
        out[i] = np.clip(np.floor((np.rint(y) + 16384) / 32768), -32768, 32767).astype(np.int16)
    return out.reshape(x.shape[:-1] + (n_out,))

