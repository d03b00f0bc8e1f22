"""The device forms of the frontend's scalar helpers on whole input domains (run with -m gpu on an H100).

mww_common.h and mww_frontend_dev.cuh give several helpers a host form and a device form (#if __CUDA_ARCH__): clz32,
shl_clamp32, mulhi_s32, vmax_u16x2, the FP64 isqrt64_round_below48 and pcm16_from_f32, and through them
wide_dynamic_function, pcan_shrink, log_scale and k2_output.  The CPU tests compile the host forms only, and the GPU parity
tests reach only the inputs their audio happens to produce.  tests/host_emul/device_forms.cu compiles the product's device
forms for sm_90a and compares them on the GPU with the portable references of tests/host_emul/scalar_refs.h (integer code
with no intrinsic form) over every input of each domain; the references are in turn tied to the oracle library on random
samples.  A failure names the first mismatching input."""

import ctypes
import os
import subprocess

import numpy as np
import pytest

import oracle
from conftest import ROOT

pytestmark = pytest.mark.gpu

HOST_EMUL = os.path.join(ROOT, "tests", "host_emul")
CSRC = os.path.join(ROOT, "microwakeword_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17"]
HARNESS_SOURCES = [os.path.join(HOST_EMUL, "device_forms.cu"), os.path.join(CSRC, "mww_tables.cc")]

WDF_PCAN, LOG_SCALE, K2_OUTPUT, ISQRT_RANGE, ISQRT_NEAR_ROOTS, PCM16, WINDOW, BITS = range(8)
NONE = (1 << 64) - 1


@pytest.fixture(scope="module")
def forms(torch_cuda, tmp_path_factory):
    so = str(tmp_path_factory.mktemp("device_forms") / "libdevice_forms.so")
    res = subprocess.run([NVCC] + NVCC_FLAGS + ["-shared", "-Xcompiler", "-fPIC", "-o", so] + HARNESS_SOURCES,
                         capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr
    L = ctypes.CDLL(so)
    u64p = ctypes.POINTER(ctypes.c_ulonglong)
    L.forms_check.argtypes = [ctypes.c_int, ctypes.c_ulonglong, ctypes.c_ulonglong, ctypes.c_void_p, ctypes.c_longlong, u64p, u64p]
    L.forms_eval.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_longlong]
    torch_cuda.cuda.init()
    assert L.forms_init() == 0
    return L


def _check(L, which, lo=0, n=0, lst=None):
    """-> (mismatches, first mismatching index or None)"""
    count, first = ctypes.c_ulonglong(0), ctypes.c_ulonglong(0)
    ptr, n_list = (lst.data_ptr(), lst.numel()) if lst is not None else (None, 0)
    assert L.forms_check(which, lo, n, ptr, n_list, ctypes.byref(count), ctypes.byref(first)) == 0
    return count.value, (None if first.value == NONE else first.value)


def _eval(torch, L, fn, x):
    """device outputs of k_eval on the uint64 inputs x (host) -> host uint32"""
    d_in = torch.from_numpy(np.ascontiguousarray(x, np.uint64).view(np.int64)).cuda()
    d_out = torch.empty(x.size, dtype=torch.int32, device="cuda")
    assert L.forms_eval(fn, d_in.data_ptr(), d_out.data_ptr(), x.size) == 0
    return d_out.cpu().numpy().view(np.uint32)


def _u32(torch, values):
    return torch.from_numpy(np.ascontiguousarray(values, np.uint32).view(np.int32)).cuda()


def test_wide_dynamic_function_and_pcan_shrink_every_uint32(forms):
    count, first = _check(forms, WDF_PCAN, 0, 1 << 32)
    assert count == 0, ("mismatches", count, "first x", first)


def test_log_scale_every_uint32_from_2(forms):
    count, first = _check(forms, LOG_SCALE, 2, (1 << 32) - 2)
    assert count == 0, ("mismatches", count, "first x", None if first is None else first + 2)


def _estimates():
    """>= 4 096 noise estimates: 0, every 2^k and 2^k +- 1, 0xFFFFFFFF, then random ones (log-uniform and uniform)"""
    rng = np.random.default_rng(20261101)
    pows = [1 << k for k in range(32)]
    fixed = sorted({v & 0xFFFFFFFF for p in pows for v in (p - 1, p, p + 1)} | {0, 0xFFFFFFFF})
    n_rand = 4096 - len(fixed)
    log_uniform = np.exp2(rng.uniform(0, 32, n_rand // 2)).astype(np.uint64)
    uniform = rng.integers(0, 1 << 32, n_rand - n_rand // 2, dtype=np.uint64)
    est = np.concatenate([np.array(fixed, np.uint64), np.minimum(log_uniform, 0xFFFFFFFF), uniform]).astype(np.uint32)
    assert est.size >= 4096
    return est


def test_k2_output_every_16_bit_value_against_4096_estimates(torch_cuda, forms):
    est = _estimates()
    count, first = _check(forms, K2_OUTPUT, lst=_u32(torch_cuda, est))
    assert count == 0, ("mismatches", count, None if first is None else ("v", first & 0xFFFF, "est", int(est[first >> 16])))


def test_isqrt_below_2_48_every_uint32(forms):
    count, first = _check(forms, ISQRT_RANGE, 0, 1 << 32)
    assert count == 0, ("mismatches", count, "first x", first)


def test_isqrt_below_2_48_next_to_every_root_below_2_24(forms):
    """n^2 - n, n^2 - n + 1 (a half-integer root between them), n^2 - 1, n^2, n^2 + n, n^2 + n + 1 for every 1 <= n < 2^24"""
    count, first = _check(forms, ISQRT_NEAR_ROOTS, 0, 6 * ((1 << 24) - 1))
    assert count == 0, ("mismatches", count, None if first is None else ("n", first // 6 + 1, "candidate", first % 6))


def test_isqrt_below_2_48_top_2_20_values(forms):
    lo = (1 << 48) - (1 << 20)
    count, first = _check(forms, ISQRT_RANGE, lo, 1 << 20)
    assert count == 0, ("mismatches", count, "first x", None if first is None else lo + first)


def test_pcm16_from_f32_every_float32_bit_pattern(forms):
    count, first = _check(forms, PCM16, 0, 1 << 32)
    assert count == 0, ("mismatches", count, "first bits", None if first is None else hex(first))


def test_window_product_every_sample_and_coefficient(forms):
    count, first = _check(forms, WINDOW)
    assert count == 0, ("mismatches", count, None if first is None else ("s", first // 4097 - 32768, "w", first % 4097))


def test_bit_helpers_edge_values_and_2_26_random_words(torch_cuda, forms):
    """clz32, msb32, shl_clamp32 for every shift 0..33, mulhi_s32 and vmax_u16x2 (both operand orders)"""
    edges = {0, 0xFFFFFFFF, 0x7FFFFFFF, 0x80000000, 0x80000001, 0x0000FFFF, 0xFFFF0000, 0x00010000, 0x7FFF7FFF, 0x80008000,
             0x8000FFFF, 0xFFFF8000, 0x00008000, 0x80000000 | 0x7FFF}
    for k in range(32):
        edges |= {((1 << k) + d) & 0xFFFFFFFF for d in (-1, 0, 1)}
        edges |= {(~(1 << k)) & 0xFFFFFFFF}
    lst = np.array(sorted(edges), np.uint32)
    count, first = _check(forms, BITS, 0, lst.size + (1 << 26), _u32(torch_cuda, lst))
    assert count == 0, ("mismatches", count, None if first is None else ("edge", hex(int(lst[first]))) if first < lst.size else ("random index", first))


# ---- the references against independent code -------------------------------------------------------------------------

def _sample_u32(rng, n, lo=0):
    """half uniform over [lo, 2^32), half log-uniform (every magnitude equally often)"""
    a = rng.integers(lo, 1 << 32, n // 2, dtype=np.uint64)
    b = np.maximum(np.exp2(rng.uniform(0, 32, n - n // 2)), lo).astype(np.uint64)
    return np.minimum(np.concatenate([a, b]), 0xFFFFFFFF)


def test_device_forms_equal_the_oracle_library_on_random_samples(torch_cuda, forms):
    """A random 2^20 sample of each device output against the oracle's C functions (mwwo_wdf, mwwo_pcan_shrink,
    mwwo_log_scaled, mwwo_sqrt64): the references above are branching restatements, this ties them to independent code."""
    O = oracle.lib()
    fe = oracle.Frontend()
    rng = np.random.default_rng(20261102)
    n = 1 << 20
    x = _sample_u32(rng, n)
    got = _eval(torch_cuda, forms, 0, x).view(np.int32)
    want = np.fromiter((O.mwwo_wdf(fe._h, int(v)) for v in x), np.int32, n)
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, ("wide_dynamic_function", int(x[bad[0]]))
    got = _eval(torch_cuda, forms, 1, x)
    want = np.fromiter((O.mwwo_pcan_shrink(int(v)) for v in x), np.uint32, n)
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, ("pcan_shrink", int(x[bad[0]]))
    x = _sample_u32(rng, n, lo=2)
    got = _eval(torch_cuda, forms, 2, x)
    want = np.fromiter((O.mwwo_log_scaled(fe._h, int(v)) for v in x), np.uint32, n)
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, ("log_scale", int(x[bad[0]]))
    x = np.concatenate([rng.integers(0, 1 << 48, n // 2, dtype=np.uint64),
                        np.exp2(rng.uniform(0, 48, n - n // 2)).astype(np.uint64)])
    x = np.minimum(x, (1 << 48) - 1)
    got = _eval(torch_cuda, forms, 3, x)
    want = np.fromiter((O.mwwo_sqrt64(int(v)) for v in x), np.uint32, n)
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, ("isqrt64_round_below48", int(x[bad[0]]))


def test_pcm16_reference_equals_to_int16_on_random_patterns(torch_cuda, forms):
    from microwakeword_b200.audio.audio_utils import to_int16
    rng = np.random.default_rng(20261103)
    bits = rng.integers(0, 1 << 32, 1 << 24, dtype=np.uint64)
    got = _eval(torch_cuda, forms, 4, bits).view(np.int32)
    with np.errstate(invalid="ignore", over="ignore"):
        want = to_int16(bits.astype(np.uint32).view(np.float32)).astype(np.int32)
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, ("float bits", hex(int(bits[bad[0]])), int(got[bad[0]]), int(want[bad[0]]))
