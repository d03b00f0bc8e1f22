"""The branch-free scalar functions of the frontend's temporal chain and windowing (mww_frontend_dev.cuh), compiled for the
CPU, equal the branching forms they replaced (kept in tests/host_emul/scalar_refs.h) on every input the kernels can
reach; and the fused clip kernels stay within 64 registers, without spills, so that four CTAs fit an SM."""

import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from conftest import ROOT

HOST_EMUL = os.path.join(ROOT, "tests", "host_emul")
CSRC = os.path.join(ROOT, "microwakeword_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


@pytest.fixture(scope="module")
def forms(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("forms") / "libemul_forms.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(HOST_EMUL, "emul_scalar_forms.cc"),
                    os.path.join(CSRC, "mww_tables.cc")], check=True)
    L = ctypes.CDLL(so)
    for name, args in (("emul_forms_wdf_pcan_mismatch", [ctypes.c_uint32, ctypes.c_uint32]),
                       ("emul_forms_log_scale_range_mismatch", [ctypes.c_uint32, ctypes.c_uint32]),
                       ("emul_forms_log_scale_list_mismatch", [ctypes.c_void_p, ctypes.c_longlong]),
                       ("emul_forms_k2_output_mismatch", [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_longlong]),
                       ("emul_forms_window_mismatch", [])):
        getattr(L, name).restype = ctypes.c_longlong
        getattr(L, name).argtypes = args
    return L


def test_wide_dynamic_function_and_pcan_shrink_on_every_uint32(forms):
    # the noise estimate is a uint32 that can take any value (the filterbank output is shifted left before smoothing), and
    # pcan_shrink's input is a uint32 product: both are checked on all 2^32 inputs
    assert forms.emul_forms_wdf_pcan_mismatch(0, 0xFFFFFFFF) == -1


def test_log_scale_below_2_24_exhaustive(forms):
    assert forms.emul_forms_log_scale_range_mismatch(2, (1 << 24) - 1) == -1


def test_log_scale_random_above_2_24(forms):
    rng = np.random.default_rng(20261016)
    x = rng.integers(1 << 24, 1 << 32, 1 << 24, dtype=np.uint64).astype(np.uint32)
    x = np.concatenate([x, np.array([1 << 24, 0xFFFFFFFF, 0x80000000, 0x7FFFFFFF], np.uint32)] +
                       [np.array([(1 << b) - 1, 1 << b, (1 << b) + 1], np.uint32) for b in range(25, 32)])
    assert forms.emul_forms_log_scale_list_mismatch(x.ctypes.data, x.size) == -1


def test_k2_output_random_pairs(forms):
    rng = np.random.default_rng(20261017)
    n = 1 << 22
    # filterbank values: mostly the usual 16-bit range, some full 32-bit; estimates over their whole range
    v = np.where(rng.random(n) < 0.9, rng.integers(0, 1 << 16, n), rng.integers(0, 1 << 32, n, dtype=np.uint64)).astype(np.uint32)
    est = np.where(rng.random(n) < 0.5, rng.integers(0, 1 << 26, n), rng.integers(0, 1 << 32, n, dtype=np.uint64)).astype(np.uint32)
    assert forms.emul_forms_k2_output_mismatch(v.ctypes.data, est.ctypes.data, n) == -1


def test_window_product_as_high_word_every_sample_and_coefficient(forms):
    assert forms.emul_forms_window_mismatch() == -1


@pytest.mark.skipif(not os.path.exists(NVCC) or shutil.which("g++") is None, reason="needs nvcc")
def test_fused_clip_kernels_fit_four_ctas_per_sm(tmp_path):
    res = subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-cubin", "-Xptxas", "-v",
                          "-o", str(tmp_path / "fe.cubin"), os.path.join(CSRC, "mww_frontend.cu")], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    regs, spills, name = {}, {}, None
    for line in res.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            name = m.group(1)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and name:
            spills[name] = int(m.group(1)) + int(m.group(2))
        m = re.search(r"Used (\d+) registers", line)
        if m and name:
            regs[name] = int(m.group(1))
    fused = [k for k in regs if "k1_spectral_kernelILb1ELi4E" in k]
    assert len(fused) == 2, sorted(regs)                  # int16 and float32 audio
    for k in fused:
        assert regs[k] <= 64 and spills[k] == 0, (k, regs[k], spills[k])


@pytest.mark.skipif(not os.path.exists(NVCC) or shutil.which("g++") is None, reason="needs nvcc")
def test_device_forms_harness_compiles_for_sm_90a(tmp_path):
    """The harness tests/test_gpu_device_forms.py runs on the GPU, compiled with the same command."""
    import test_gpu_device_forms as T
    res = subprocess.run([NVCC] + T.NVCC_FLAGS + ["-shared", "-Xcompiler", "-fPIC", "-o", str(tmp_path / "forms.so")] + T.HARNESS_SOURCES,
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
