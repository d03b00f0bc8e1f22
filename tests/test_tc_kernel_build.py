"""The wgmma clip kernel (mww_nn_tc.cu) compiles for sm_90a within the register budget of its planned occupancy -- two CTAs of
256 threads per SM, so at most 128 registers a thread -- without spills, and its contractions are HGMMA instructions."""

import os
import re
import shutil
import subprocess

import pytest

from conftest import ROOT

CSRC = os.path.join(ROOT, "microwakeword_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
KERNEL = "nn_f32_clip_tc_kernel"


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    if not os.path.exists(NVCC) or shutil.which("g++") is None:
        pytest.skip("needs nvcc")
    cubin = str(tmp_path_factory.mktemp("tc") / "tc.cubin")
    res = subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-cubin", "-Xptxas", "-v",
                          "-o", cubin, os.path.join(CSRC, "mww_nn_tc.cu")], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    return res.stderr, cubin


def test_tc_kernel_fits_two_ctas_per_sm_without_spills(compiled):
    log, _ = compiled
    name, info = None, {}
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            name = m.group(1)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and name and KERNEL in name:
            info["spill"] = int(m.group(1)) + int(m.group(2))
        m = re.search(r"Used (\d+) registers", line)
        if m and name and KERNEL in name:
            info["regs"] = int(m.group(1))
    assert set(info) == {"spill", "regs"}, log
    assert info["regs"] <= 65536 // (2 * 256) and info["spill"] == 0, info


def test_tc_kernel_contracts_on_hgmma(compiled):
    _, cubin = compiled
    cuobjdump = os.path.join(os.path.dirname(NVCC), "cuobjdump")
    sass = subprocess.run([cuobjdump, "-sass", cubin], capture_output=True, text=True).stdout
    body = sass.split(KERNEL, 1)
    assert len(body) == 2, "kernel missing from the cubin"
    assert "HGMMA" in body[1].split("Function :", 1)[0]
