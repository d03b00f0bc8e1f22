"""The float32 -> int16 sample conversion of the frontend kernels (pcm16_from_f32, mww_frontend_dev.cuh), compiled for the
CPU, equals the host rule audio_utils.to_int16 -- np.clip(x * 32768, -32768, 32767).astype(np.int16), the reference's
conversion of float clips -- on every float32 near an integer boundary, on the IEEE special values and on 2^24 random bit
patterns."""

import ctypes
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from microwakeword_b200.audio.audio_utils import to_int16

HOST_EMUL = os.path.join(ROOT, "tests", "host_emul")


@pytest.fixture(scope="module")
def convert(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("pcm16") / "libemul_pcm16.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(HOST_EMUL, "emul_pcm16.cc")], check=True)
    fn = ctypes.CDLL(so).emul_pcm16_from_f32
    fn.restype = None
    fn.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_longlong]

    def run(x):
        x = np.ascontiguousarray(x, np.float32)
        out = np.empty(x.shape, np.int16)
        fn(x.ctypes.data, out.ctypes.data, x.size)
        return out
    return run


def _host(x):
    with np.errstate(invalid="ignore", over="ignore"):     # NaN / inf and x * 32768 overflow warn in numpy; their results are what is compared
        return to_int16(np.asarray(x, np.float32))


def _f32(bits):
    return np.asarray(bits, np.uint32).view(np.float32)


def test_every_float_within_two_ulp_of_each_integer_boundary(convert):
    k = np.arange(-32770, 32771)
    centre = (k / 32768.0).astype(np.float32)            # exact: k / 2^15 with |k| < 2^24
    xs = [centre]
    for direction in (np.inf, -np.inf):
        x = centre
        for _ in range(2):
            x = np.nextafter(x, np.float32(direction))
            xs.append(x)
    x = np.concatenate(xs)
    assert x.size == 5 * k.size
    assert np.array_equal(convert(x), _host(x))


def test_special_values(convert):
    nans = _f32([0x7FC00000, 0xFFC00000, 0x7F800001, 0xFF800001, 0x7FA5A5A5, 0x7FFFFFFF, 0xFFFFFFFF])
    subnormals = _f32([0x00000001, 0x80000001, 0x00400000, 0x007FFFFF, 0x807FFFFF])
    flt_max = np.finfo(np.float32).max
    x = np.concatenate([np.array([0.0, -0.0, np.inf, -np.inf, flt_max, -flt_max], np.float32), nans, subnormals,
                        np.array([0.99999994, 3.0517578e-05, -3.0517578e-05, 1.0, -1.0, 1.5, -1.5], np.float32)])
    got = convert(x)
    assert np.array_equal(got, _host(x))
    # the rule spelled out, independent of numpy: +-0 -> 0, +-inf and +-FLT_MAX clamp, NaN -> 0, subnormals -> 0
    want = [0, 0, 32767, -32768, 32767, -32768] + [0] * nans.size + [0] * subnormals.size + [32767, 1, -1, 32767, -32768, 32767, -32768]
    assert got.tolist() == want


def test_random_bit_patterns(convert):
    rng = np.random.default_rng(20261015)
    x = rng.integers(0, 2 ** 32, 2 ** 24, dtype=np.uint64).astype(np.uint32).view(np.float32)
    got, want = convert(x), _host(x)
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, [(hex(int(x[i:i + 1].view(np.uint32)[0])), int(got[i]), int(want[i])) for i in bad[:8]]
