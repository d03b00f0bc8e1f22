"""The fused clip frontend k1_clip_kernel (microwakeword_b200/csrc/mww_frontend_clip.cu, companion library
libmww_frontend_clip.so), the parts that need no GPU:

  * its group schedule emulated on the CPU (tests/emul_frontend_clip.cc, built with g++ over the product's phase functions):
    only __syncwarp between the phases from the window to the filterbank, run warp after warp in both orders, and the next
    group's audio loaded before this group's pass 1 -- features, estimate and carry against the oracle and the emulation of
    the separate K1 + K2 kernels, over several calls that carry state;
  * the library: exactly its kernels (four sample types, each with the vector and the per-sample loaders), 64 registers or
    fewer, no stack, local memory or spills, shared memory for four CTAs per SM; libmww_b200.so needs it and the build knows
    it is missing."""

import ctypes
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

import oracle
from conftest import ROOT, edge_case_audio, synth_audio
from host_emul import emul as host_emul

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(ROOT, "microwakeword_b200", "csrc")
_BUILD = tempfile.TemporaryDirectory(prefix="mww_frontend_clip_test_")
_emul = []
vp, i32 = ctypes.c_void_p, ctypes.c_int


def emul():
    if not _emul:
        so = os.path.join(_BUILD.name, "libemul_frontend_clip.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "emul_frontend_clip.cc"),
                        os.path.join(CSRC, "mww_tables.cc")], check=True)
        L = ctypes.CDLL(so)
        L.emul_clip_features.restype = i32
        L.emul_clip_features.argtypes = [vp, i32, i32, vp, i32, vp, vp, i32, ctypes.POINTER(i32), i32]
        L.emul_k1_smem_bytes.restype = i32
        _emul.append(L)
    return _emul[0]


def _p(a):
    return ctypes.c_void_p(a.ctypes.data)


class ClipFrontend:
    """the emulated kernel's call sequence for S lockstep streams"""

    def __init__(self, n_streams, order):
        self.carry = np.zeros((n_streams, 480), np.int16)
        self.estimate = np.zeros((n_streams, 40), np.uint32)
        self.used, self.order = 0, order

    def features(self, audio):
        audio = np.ascontiguousarray(audio, np.int16)
        S, N = audio.shape
        rows = (self.used + N) // 160 + 1
        feat = np.zeros((S, rows, 40), np.uint16)
        nu = i32(0)
        n = emul().emul_clip_features(_p(audio), S, N, _p(self.carry), self.used, _p(self.estimate), _p(feat), rows, ctypes.byref(nu),
                                      self.order)
        assert n >= 0
        self.used = nu.value
        return feat[:, :n]


def _audio(n):
    rng = np.random.default_rng(11)
    rows = [synth_audio(n, 300 + i) for i in range(4)] + [e[:n] for e in edge_case_audio(n)[:5]]
    rows.append(rng.choice([-32768, 32767], n).astype(np.int16))
    rows.append(np.clip(np.round(rng.normal(0, 20000, n)), -32768, 32767).astype(np.int16))
    return np.stack(rows)


CALLS = (4000, 1760, 6400, 3840)          # 24, 11, 40 and 24 frames: ragged last groups, 320 samples carried in and out


@pytest.mark.parametrize("order", [0, 1])
def test_half_warp_schedule_matches_the_oracle(order):
    """11 streams, four calls carrying carry, used and estimate.  Features equal the oracle's, and state equals that of the
    emulated separate K1 + K2 kernels after every call."""
    audio = _audio(sum(CALLS))
    want, _ = oracle.run_pipeline(None, audio, want_probs=False)
    fe, sep = ClipFrontend(audio.shape[0], order), host_emul.Frontend(audio.shape[0])
    pos, got = 0, []
    for n in CALLS:
        got.append(fe.features(audio[:, pos:pos + n]))
        sep.features(audio[:, pos:pos + n])
        assert fe.used == sep.used and np.array_equal(fe.estimate, sep.estimate) and np.array_equal(fe.carry, sep.carry), (order, n)
        pos += n
    got = np.concatenate(got, 1)
    assert got.shape == want.shape and np.array_equal(got, want), order


def _cuobjdump():
    from microwakeword_b200 import _lib, build
    tool = os.path.join(os.path.dirname(build.NVCC), "cuobjdump")
    if not os.path.exists(tool):
        pytest.skip("cuobjdump is not installed next to nvcc")
    _lib.lib()
    return tool


def test_companion_library_holds_exactly_its_kernels_within_four_ctas_per_sm(monkeypatch):
    from microwakeword_b200 import build
    assert os.path.basename(build.FC_OUT) == "libmww_frontend_clip.so" and build.FC_SOURCES == ["mww_frontend_clip.cu"]
    res = subprocess.run([_cuobjdump(), "-res-usage", build.FC_OUT], capture_output=True, text=True, check=True).stdout
    found = re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", res)
    names = sorted(n for n, *_ in found)
    want = sorted("_ZN3mww14k1_clip_kernelI%sLb%dEEEvNS_14FrontendParamsEPKsiPKT_xiiPjPtx" % (t, v)
                  for t in ("s", "f", "NS_5Ulaw8E", "NS_5Alaw8E") for v in (0, 1))
    assert names == want, res
    smem = emul().emul_k1_smem_bytes()
    for name, reg, stack, shared, local in found:
        assert int(reg) <= 64 and int(stack) == 0 and int(local) == 0, (name, reg, stack, local)
        # SHARED is the 1 KB the H100 reserves per CTA: the kernel declares no static shared memory of its own
        assert int(shared) <= 1024 and 4 * (int(shared) + smem) <= 228 * 1024, (name, shared, smem)
    flags = [f for f in build.FLAGS if f not in ("-shared", "-cudart", "static")]
    rep = subprocess.run([build.NVCC] + flags + ["-cubin", "-Xptxas", "-v", "-o", os.path.join(_BUILD.name, "clip.cubin"),
                                                 os.path.join(CSRC, "mww_frontend_clip.cu")], capture_output=True, text=True, check=True).stderr
    spills = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", rep)
    assert len(spills) == 8 and all(int(a) == int(b) == int(c) == 0 for a, b, c in spills), rep
    dyn = subprocess.run(["readelf", "-d", build.OUT], capture_output=True, text=True).stdout
    assert "[libmww_frontend_clip.so]" in dyn
    real = os.path.exists
    monkeypatch.setattr(build.os.path, "exists", lambda p: p != build.FC_OUT and real(p))
    assert build._stale()
