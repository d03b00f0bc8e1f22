"""G.711 audio without a GPU: the decode the kernels apply (a g++ build of mww_frontend_dev.cuh) on all 256 codes of each
law against the rule stated in include/mww.h and against Python's audioop; the seven _g711 entry points in the header, the
export list and the binding; the Python refusals that run before the library is called; the companion library
libmww_g711.so, its kernels and their register use; and the timing tool's loud failure without a GPU."""

import ctypes
import os
import re
import shutil
import subprocess
import sys
import warnings

import numpy as np
import pytest

from conftest import ROOT

HOST_EMUL = os.path.join(ROOT, "tests", "host_emul")
G711_FORMS = {
    "mww_features_g711": "mww_features",
    "mww_predict_clip_g711": "mww_predict_clip",
    "mww_predict_clip_host_g711": "mww_predict_clip_host",
    "mww_predict_clip_remote_g711": "mww_predict_clip_remote",
    "mww_predict_clip_multi_g711": "mww_predict_clip_multi",
    "mww_predict_clip_host_multi_g711": "mww_predict_clip_host_multi",
    "mww_predict_clip_remote_multi_g711": "mww_predict_clip_remote_multi",
}
CODES = np.arange(256, dtype=np.uint8)


# ---- the decode rule ---------------------------------------------------------------------------------------------------
def ulaw_ref(code):
    """include/mww.h's mu-law rule, restated in NumPy"""
    u = (~np.asarray(code, np.int64)) & 0xFF
    t = (((u & 0x0F) << 3) + 0x84) << ((u & 0x70) >> 4)
    return np.where(u & 0x80, 0x84 - t, t - 0x84).astype(np.int16)


def alaw_ref(code):
    """include/mww.h's A-law rule, restated in NumPy"""
    a = np.asarray(code, np.int64) ^ 0x55
    t = (a & 0x0F) << 4
    seg = (a & 0x70) >> 4
    t = np.where(seg == 0, t + 8, np.where(seg == 1, t + 0x108, (t + 0x108) << np.maximum(seg - 1, 0)))
    return np.where(a & 0x80, t, -t).astype(np.int16)


@pytest.fixture(scope="module")
def decode(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("g711") / "libemul_g711.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(HOST_EMUL, "emul_g711.cc")], check=True)
    fn = ctypes.CDLL(so).emul_g711_decode
    fn.restype = None
    fn.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_longlong]

    def run(law, codes):
        codes = np.ascontiguousarray(codes, np.uint8)
        out = np.empty(codes.shape, np.int16)
        fn(law, codes.ctypes.data, out.ctypes.data, codes.size)
        return out
    return run


def test_kernel_decode_matches_the_stated_rule(decode):
    assert np.array_equal(decode(1, CODES), ulaw_ref(CODES))
    assert np.array_equal(decode(2, CODES), alaw_ref(CODES))


def test_kernel_decode_matches_audioop(decode):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", DeprecationWarning)
        audioop = pytest.importorskip("audioop")
    ulaw = np.frombuffer(audioop.ulaw2lin(CODES.tobytes(), 2), "<i2")
    alaw = np.frombuffer(audioop.alaw2lin(CODES.tobytes(), 2), "<i2")
    assert np.array_equal(decode(1, CODES), ulaw)
    assert np.array_equal(decode(2, CODES), alaw)


def test_spot_values_and_ranges(decode):
    u, a = decode(1, CODES), decode(2, CODES)
    assert (u[0x00], u[0x80], u[0xFF], u[0x7F]) == (-32124, 32124, 0, 0)
    assert (a[0xD5], a[0x55], a[0xAA], a[0x2A]) == (8, -8, 32256, -32256)
    assert u.min() == -32124 and u.max() == 32124 and a.min() == -32256 and a.max() == 32256
    assert np.unique(u).size == 255 and np.unique(a).size == 256      # mu-law has two zeros, A-law none


# ---- C-ABI and binding ---------------------------------------------------------------------------------------------------
def _header():
    return open(os.path.join(ROOT, "include", "mww.h")).read()


def test_entry_points_declared_exported_and_bound():
    from microwakeword_b200 import _lib
    L = _lib.lib()
    hdr = _header()
    for name, int16_form in G711_FORMS.items():
        assert name in _lib.EXPORTS and hasattr(L, name), name
        fn, ref = getattr(L, name), getattr(L, int16_form)
        assert fn.restype is ctypes.c_int
        assert fn.argtypes == ref.argtypes[:2] + [ctypes.c_int] + ref.argtypes[2:], name
        decl = re.search(r"int %s\(mww_t \*h, const (\w+) \*\w+, int law," % name, hdr)
        assert decl and decl.group(1) == "uint8_t", name


def test_law_constants_in_header_and_binding():
    from microwakeword_b200 import _lib
    hdr = _header()
    assert re.search(r"#define MWW_G711_ULAW 1\b", hdr) and re.search(r"#define MWW_G711_ALAW 2\b", hdr)
    assert (_lib.MWW_G711_ULAW, _lib.MWW_G711_ALAW) == (1, 2)


# ---- Python refusals before the library --------------------------------------------------------------------------------
def _engine(cls, n_streams=4):
    """an engine object with no handle: enough for the checks that run before the library is called"""
    from microwakeword_b200 import _lib
    e = object.__new__(cls)
    e._L, e._h, e.n_streams = _lib.lib(), None, n_streams
    return e


def test_host_audio_law_pairing():
    from microwakeword_b200.engine import MultiModelEngine, StreamEngine
    for cls in (StreamEngine, MultiModelEngine):
        e = _engine(cls)
        codes = np.zeros((4, 480), np.uint8)
        for law in ("ulaw", "alaw"):
            a, pitch, is_f32 = e._check_host_audio(codes[:, 3:483 - 8], law=law)      # a column slice keeps its pitch
            assert np.shares_memory(a, codes) and pitch == 480 and not is_f32
        for audio, law in ((codes, None), (np.zeros((4, 480), np.int16), "ulaw"), (np.zeros((4, 480), np.float32), "alaw"),
                           (codes, "pcmu"), (codes, "ULAW"), (codes, 1), (np.zeros((4, 480), np.int8), "ulaw")):
            with pytest.raises(ValueError):
                e._check_host_audio(audio, law=law)
        with pytest.raises(ValueError):
            e.predict_clip_host(codes)                             # uint8 without a law: refused before the library
        with pytest.raises(ValueError):
            e.predict_clip_host(codes, law="mulaw")


def test_remote_law_selects_the_g711_entry_point():
    import torch
    from microwakeword_b200 import _lib
    from microwakeword_b200.engine import MultiModelEngine, StreamEngine
    calls = []

    class Recorder:
        def __init__(self, name):
            self.name = name

        def __call__(self, *args):
            calls.append((self.name, args))
            return 0

    for cls, name in ((StreamEngine, "mww_predict_clip_remote"), (MultiModelEngine, "mww_predict_clip_remote_multi")):
        e = _engine(cls)
        L = e._L
        assert e._remote_fn(np.int16, name) is getattr(L, name)
        assert e._remote_fn(np.float32, name) is getattr(L, name + "_f32")
        for dt in (np.uint8, "uint8", torch.uint8):
            for law, code in (("ulaw", _lib.MWW_G711_ULAW), ("alaw", _lib.MWW_G711_ALAW)):
                calls.clear()
                e._L = type("L", (), {name + "_g711": Recorder(name + "_g711")})()
                fn = e._remote_fn(dt, name, law)
                fn("h", "ptr", 480, 480)
                assert calls == [(name + "_g711", ("h", "ptr", code, 480, 480))]
                e._L = L
        for dt, law in ((np.uint8, None), (np.int16, "ulaw"), (np.float32, "alaw"), (np.uint8, "g722"), (np.uint16, "ulaw")):
            with pytest.raises(ValueError):
                e._remote_fn(dt, name, law)
        with pytest.raises(ValueError):                        # refused before any device work
            e.predict_clip_remote(0, 480, dtype=np.uint8)
        with pytest.raises(ValueError):
            e.predict_clip_remote(0, 480, dtype=np.int16, law="ulaw")


# ---- the companion library -----------------------------------------------------------------------------------------------
def _cuobjdump():
    from microwakeword_b200 import _lib, build
    tool = os.path.join(os.path.dirname(build.NVCC), "cuobjdump")
    if not os.path.exists(tool):
        pytest.skip("cuobjdump is not installed next to nvcc")
    _lib.lib()
    return tool


def test_library_is_built_and_linked():
    from microwakeword_b200 import _lib, build
    _lib.lib()
    assert os.path.exists(build.G711_OUT)
    if shutil.which("readelf"):
        dyn = subprocess.run(["readelf", "-d", build.OUT], capture_output=True, text=True, check=True).stdout
        assert "[libmww_g711.so]" in dyn and "$ORIGIN" in dyn


def test_every_kernel_reads_g711_and_none_spills():
    from microwakeword_b200 import build
    res = subprocess.run([_cuobjdump(), "-res-usage", build.G711_OUT], capture_output=True, text=True, check=True).stdout
    found = re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", res)
    # five frontend launchers (seven kernels: the clip kernel in three forms) and two resampler forms, per law
    assert len(found) == 18, res[-2000:]
    for law in ("Ulaw8", "Alaw8"):
        assert sum(law in name for name, *_ in found) == 9
    for name, reg, stack, local in found:
        assert "Ulaw8" in name or "Alaw8" in name, name
        assert int(stack) == 0 and int(local) == 0, name


def test_timing_tool_fails_loudly_without_a_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present; the loud-failure path is exercised on GPU-less hosts")
    tool = os.path.join(ROOT, "tools", "g711_time.py")
    res = subprocess.run([sys.executable, tool, "--streams", "64"], capture_output=True, text=True)
    assert res.returncode != 0 and "CUDA" in res.stderr
