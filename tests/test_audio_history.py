"""The audio history without a GPU: the ring index math and the append / read kernel bodies (a g++ build of
microwakeword_b200/csrc/mww_history.h, tests/emul_history.cc) against a NumPy model of the rule in include/mww.h (zeros, then
every sample appended since the last zeroing; a read returns the last n); the four entry points in the header, the export
list and the binding; the Python refusals that run before the library is called; the companion library libmww_history.so,
its kernels and their register use; and the timing tool's loud failure without a GPU."""

import ctypes
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT

HERE = os.path.dirname(os.path.abspath(__file__))
ENTRY_POINTS = ("mww_set_audio_history", "mww_get_audio_history", "mww_read_audio_history", "mww_read_audio_history_device_ids")


def _p(a):
    return ctypes.c_void_p(a.ctypes.data)


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("history") / "libemul_history.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "emul_history.cc")], check=True)
    L = ctypes.CDLL(so)
    L.emul_history_capacity_ok.argtypes = [ctypes.c_longlong]
    L.emul_history_append.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_longlong, ctypes.c_void_p,
                                      ctypes.c_longlong, ctypes.c_int, ctypes.c_int]
    L.emul_history_read.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_longlong, ctypes.c_void_p, ctypes.c_int,
                                    ctypes.c_int, ctypes.c_void_p, ctypes.c_longlong]
    return L


class Model:
    """The rule: each stream's history is zeros followed by every sample appended since it was last zeroed."""

    def __init__(self, n_streams):
        self.runs = [np.zeros(0, np.int16) for _ in range(n_streams)]

    def append(self, samples):                   # [n_streams, n16] int16
        self.runs = [np.concatenate([r, s]) for r, s in zip(self.runs, samples)]

    def zero(self, ids):
        for i in ids:
            self.runs[i] = np.zeros(0, np.int16)

    def read(self, ids, n):
        out = np.zeros((len(ids), n), np.int16)
        for j, i in enumerate(ids):
            if 0 <= i < len(self.runs) and n:
                tail = self.runs[i][-n:]
                out[j, n - tail.size:] = tail
        return out


class Ring:
    """The kernels' ring and lockstep counter, driven through the g++ build of their bodies"""

    def __init__(self, emul, n_streams, C):
        self.L, self.S, self.C, self.seen = emul, n_streams, C, 0
        self.ring = np.zeros((n_streams, C), np.int16)

    def append(self, audio, type_=0, allow_vec=1, stride=None, n16=None):
        n16 = audio.shape[1] if n16 is None else n16
        stride = audio.strides[0] // audio.itemsize if stride is None else stride
        vec = self.L.emul_history_append(type_, _p(self.ring), self.S, self.C, self.seen, _p(audio), stride, n16, allow_vec)
        self.seen += n16
        return vec

    def zero(self, ids):
        self.ring[list(ids)] = 0

    def read(self, ids, n, pad=0):
        ids = np.ascontiguousarray(ids, np.int32)
        out = np.full((ids.size, n + pad), 7, np.int16)
        vec = self.L.emul_history_read(_p(self.ring), self.C, self.S, self.seen, _p(ids), ids.size, n, _p(out), n + pad)
        assert (out[:, n:] == 7).all()           # nothing written past n_samples
        return out[:, :n], vec


def test_capacities(emul):
    for C in (0, 8, 16, 480, 32000, 1 << 22):
        assert emul.emul_history_capacity_ok(C)
    for C in (-8, 1, 4, 7, 12, 481, (1 << 22) + 8, 1 << 23):
        assert not emul.emul_history_capacity_ok(C)


@pytest.mark.parametrize("C", [8, 480, 32000])
def test_random_calls_zeroing_and_reads_match_the_rule(emul, C):
    rng = np.random.default_rng(C)
    S = 5
    ring, model = Ring(emul, S, C), Model(S)
    lengths = [16, 0, 1, 7, 161, 480, C + 3, 8, 16, 2 * C + 8, 3] + list(rng.integers(0, 3 * C + 17, 12))
    vec_seen = set()
    for t, n16 in enumerate(lengths):
        audio = rng.integers(-32768, 32768, (S, int(n16)), dtype=np.int64).astype(np.int16)
        vec_seen.add(ring.append(audio))
        model.append(audio)
        if t % 4 == 3:                            # zero some rows, or all
            ids = list(range(S)) if t % 8 == 7 else [1, 3]
            ring.zero(ids)
            model.zero(ids)
        for n in (0, 1, C, min(C, 9), min(C, 24)):
            ids = [0, 4, 2, 2, 1]
            got, _ = ring.read(ids, n)
            assert np.array_equal(got, model.read(ids, n)), (C, t, n)
    assert ring.seen > 3 * C                      # many wraps
    assert vec_seen == {0, 1}                     # both forms ran


def test_vector_and_scalar_forms_agree(emul):
    """the same calls through the 8-sample units (where the shape allows) and through single samples"""
    rng = np.random.default_rng(1)
    C = 64
    a, b, model = Ring(emul, 3, C), Ring(emul, 3, C), Model(3)
    for n16 in (8, 16, 24, 7, 9, 40, 64, 72, 200, 8):
        audio = rng.integers(-32768, 32768, (3, n16), dtype=np.int64).astype(np.int16)
        a.append(audio, allow_vec=1)
        b.append(audio, allow_vec=0)
        model.append(audio)
        assert np.array_equal(a.ring, b.ring)
        for n in (8, 16, 64, 5):
            assert np.array_equal(a.read([0, 1, 2], n)[0], model.read([0, 1, 2], n))


def test_vector_shape_conditions(emul):
    audio = np.zeros((2, 64), np.int16)
    r = Ring(emul, 2, 32)
    assert r.append(audio[:, :16]) == 1                 # slot 0, source 0, 16 samples, pitch 64
    assert r.append(audio[:, :7]) == 0                  # m % 8 != 0
    assert r.append(audio[:, :16]) == 0                 # now the slot is 23
    r = Ring(emul, 2, 32)
    assert r.append(audio[:, :40]) == 1                 # longer than C: source starts at 8, slot 8
    assert r.append(audio[:, :36]) == 0                 # source starts at 4
    r = Ring(emul, 2, 32)
    assert r.append(audio[:, :16], stride=60) == 0      # pitch % 8 != 0
    _, vec = r.read([0, 1], 16)
    assert vec == 1
    _, vec = r.read([0, 1], 12)
    assert vec == 0


@pytest.mark.parametrize("type_", [1, 2, 3])
def test_other_sample_types_append_their_int16_samples(emul, type_):
    """float32 appends the converted samples, G.711 the decoded ones (the pcm16 overloads of the frontend)"""
    from test_g711 import alaw_ref, ulaw_ref
    rng = np.random.default_rng(type_)
    C = 48
    r, model = Ring(emul, 2, C), Model(2)
    for n16 in (16, 5, 40, 64, 3):
        if type_ == 1:
            audio = (rng.standard_normal((2, n16)) * 0.6).astype(np.float32)
            audio[0, :2] = (np.nan, 1.5) if n16 >= 2 else audio[0, :2]
            want = np.clip(audio.astype(np.float32) * 32768, -32768, 32767)
            want = np.where(np.isnan(want), 0, want).astype(np.int16)
        else:
            audio = rng.integers(0, 256, (2, n16), dtype=np.int64).astype(np.uint8)
            want = ulaw_ref(audio) if type_ == 2 else alaw_ref(audio)
        r.append(audio, type_=type_)
        model.append(want)
        assert np.array_equal(r.read([0, 1], C)[0], model.read([0, 1], C))


def test_device_id_reads_give_zero_rows_for_out_of_range_ids(emul):
    rng = np.random.default_rng(5)
    r, model = Ring(emul, 4, 16), Model(4)
    audio = rng.integers(-30000, 30000, (4, 24), dtype=np.int64).astype(np.int16)
    r.append(audio)
    model.append(audio)
    ids = [-1, 3, 4, 0, -1, 3, 1 << 20]
    got, _ = r.read(ids, 16)
    assert np.array_equal(got, model.read(ids, 16))
    assert (got[[0, 2, 4, 6]] == 0).all() and np.array_equal(got[1], audio[3, -16:])


# ---- C-ABI and binding ---------------------------------------------------------------------------------------------------
def test_entry_points_declared_exported_and_bound():
    from microwakeword_b200 import _lib
    L = _lib.lib()
    hdr = open(os.path.join(ROOT, "include", "mww.h")).read()
    for name in ENTRY_POINTS:
        assert name in _lib.EXPORTS and hasattr(L, name), name
        assert getattr(L, name).restype is ctypes.c_int
    vp, i32, ll = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong
    assert L.mww_set_audio_history.argtypes == [vp, i32, vp]
    assert L.mww_get_audio_history.argtypes == [vp, ctypes.POINTER(i32), ctypes.POINTER(ll)]
    for name in ENTRY_POINTS[2:]:
        assert getattr(L, name).argtypes == [vp, vp, i32, i32, vp, ll, vp], name
    assert re.search(r"int mww_set_audio_history\(mww_t \*h, int capacity, void \*cu_stream\);", hdr)
    assert re.search(r"int mww_get_audio_history\(const mww_t \*h, int \*capacity, long long \*samples_seen\);", hdr)
    assert re.search(r"int mww_read_audio_history\(mww_t \*h, const int32_t \*h_ids, int n, int n_samples, int16_t \*d_out, "
                     r"long long out_stride, void \*cu_stream\);", hdr)
    assert re.search(r"int mww_read_audio_history_device_ids\(mww_t \*h, const int32_t \*d_ids, int n, int n_samples, int16_t \*d_out, "
                     r"long long out_stride,\s+void \*cu_stream\);", hdr)


def test_null_handle_is_refused():
    from microwakeword_b200 import _lib
    L = _lib.lib()
    assert L.mww_set_audio_history(None, 8, None) == -1
    assert L.mww_get_audio_history(None, None, None) == -1
    assert L.mww_read_audio_history(None, None, 0, 0, None, 0, None) == -1
    assert L.mww_read_audio_history_device_ids(None, None, 0, 0, None, 0, None) == -1


# ---- Python refusals before the library --------------------------------------------------------------------------------
class _Refusing:
    """stands in for the library: every call fails the test, so a refusal must come from Python"""

    def __init__(self, capacity=32):
        self.capacity = capacity

    def mww_get_audio_history(self, h, cap, seen):
        cap._obj.value = self.capacity
        return 0

    def __getattr__(self, name):
        raise AssertionError("the library was called: " + name)


def _engine(cls, capacity=32, n_streams=4):
    e = object.__new__(cls)
    e._L, e._h, e.n_streams, e.device = _Refusing(capacity), None, n_streams, 0
    return e


def test_python_refusals():
    from microwakeword_b200.engine import MultiModelEngine, StreamEngine
    for cls in (StreamEngine, MultiModelEngine):
        e = _engine(cls)
        for bad in (-8, 1, 4, 12, 481, (1 << 22) + 8, 1 << 23, 8.5, True, "32"):
            with pytest.raises((ValueError, TypeError)):
                e.set_audio_history(bad)
        for n in (-1, 33, 2.5, True):
            with pytest.raises(ValueError):
                e.audio_history([0, 1], n)
        for ids in ([0, 4], [-1], [[0, 1]], [0.5], np.array([[1]])):
            with pytest.raises(ValueError):
                e.audio_history(ids, 8)
        with pytest.raises(ValueError):
            _engine(cls, capacity=0).audio_history([0], 0)          # no history


def test_python_refusals_of_tensor_arguments():
    torch = pytest.importorskip("torch")
    from microwakeword_b200.engine import StreamEngine
    e = _engine(StreamEngine)
    with pytest.raises(ValueError):
        e.audio_history(torch.zeros((2, 2), dtype=torch.int32), 8)     # a CPU tensor is a host list, and this one is 2-D
    for out in (np.zeros((2, 8), np.int16), torch.zeros((2, 8), dtype=torch.int16)):
        with pytest.raises(ValueError):
            e.audio_history([0, 1], 8, out=out)                       # not device memory


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
    assert os.path.exists(build.HIST_OUT)
    if shutil.which("readelf"):
        dyn = subprocess.run(["readelf", "-d", build.OUT], capture_output=True, text=True, check=True).stdout
        assert "[libmww_history.so]" in dyn and "$ORIGIN" in dyn


def test_kernel_set_and_no_spills():
    from microwakeword_b200 import build
    res = subprocess.run([_cuobjdump(), "-res-usage", build.HIST_OUT], capture_output=True, text=True, check=True).stdout
    found = re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", res)
    names = sorted(name for name, *_ in found)
    assert len(found) == 5, res[-2000:]
    assert sum("history_read_kernel" in n for n in names) == 1
    for t in ("IsE", "IfE", "INS_5Ulaw8EE", "INS_5Alaw8EE"):          # int16, float, mu-law, A-law
        assert sum("history_append_kernel" + t in n for n in names) == 1, (t, names)
    for name, reg, stack, local in found:
        assert int(stack) == 0 and int(local) == 0, name


def test_main_library_does_not_hold_the_history_kernels():
    from microwakeword_b200 import build
    res = subprocess.run([_cuobjdump(), "-res-usage", build.OUT], capture_output=True, text=True, check=True).stdout
    assert "history_" not in res


def test_timing_tool_fails_loudly_without_a_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present; the loud-failure path is exercised on GPU-less hosts")
    tool = os.path.join(ROOT, "tools", "audio_history_time.py")
    res = subprocess.run([sys.executable, tool, "--streams", "64"], capture_output=True, text=True)
    assert res.returncode != 0 and "CUDA" in res.stderr
