"""The float32 host / remote entry points without a GPU: the library exports them, the binding declares them with the
argument lists of their int16 counterparts, and the Python argument checks that need no device."""

import ctypes
import os
import re

import numpy as np
import pytest

from conftest import ROOT

FLOAT_FORMS = {
    "mww_predict_clip_host_f32": "mww_predict_clip_host",
    "mww_predict_clip_host_multi_f32": "mww_predict_clip_host_multi",
    "mww_predict_clip_remote_f32": "mww_predict_clip_remote",
    "mww_predict_clip_remote_multi_f32": "mww_predict_clip_remote_multi",
}


def test_float_forms_are_exported_and_declared_like_their_int16_counterparts():
    from microwakeword_b200 import _lib
    L = _lib.lib()
    hdr = open(os.path.join(ROOT, "include", "mww.h")).read()
    for name, int16_form in FLOAT_FORMS.items():
        assert name in _lib.EXPORTS and hasattr(L, name), name
        fn, ref = getattr(L, name), getattr(L, int16_form)
        assert fn.restype is ctypes.c_int and fn.argtypes == ref.argtypes, name
        decl = re.search(r"int %s\(mww_t \*h, const (\w+) \*\w+," % name, hdr)
        assert decl and decl.group(1) == "float", name


def _engine(cls, n_streams=4):
    """an engine object with no handle: enough for the checks that run before the library is called"""
    from microwakeword_b200 import _lib
    e = object.__new__(cls)
    e._L, e._h, e.n_streams = _lib.lib(), None, n_streams
    return e


@pytest.mark.parametrize("dtype", [np.int16, np.float32])
def test_host_audio_check_accepts_int16_and_float32(dtype):
    from microwakeword_b200.engine import StreamEngine
    e = _engine(StreamEngine)
    wide = np.zeros((4, 500), dtype)
    a, pitch, is_f32 = e._check_host_audio(wide[:, 7:487])               # a column slice keeps its row pitch, no copy
    assert np.shares_memory(a, wide) and pitch == 500 and is_f32 == (dtype == np.float32)
    a, pitch, _ = e._check_host_audio(wide[:, ::2])                       # samples not contiguous: copied
    assert not np.shares_memory(a, wide) and a.flags.c_contiguous and pitch == 250
    a, pitch, _ = e._check_host_audio(np.zeros((4, 0), dtype))
    assert pitch == 0


@pytest.mark.parametrize("dtype", [np.int16, np.float32])
def test_host_audio_check_copies_row_strides_the_library_cannot_express(dtype):
    """a row stride that is not a whole number of samples, or is below n_samples (broadcast, reversed rows), would make the
    library read the wrong samples or refuse the call: such arrays are copied, values unchanged"""
    from numpy.lib.stride_tricks import as_strided
    from microwakeword_b200.engine import StreamEngine
    e = _engine(StreamEngine)
    size = np.dtype(dtype).itemsize
    raw = np.zeros(4 * (480 * size + 1) + 480 * size, np.uint8)
    raw[:] = np.arange(raw.size) % 251
    odd = as_strided(raw[:480 * size].view(dtype), shape=(4, 480), strides=(480 * size + 1, size))
    odd_values = np.array([raw[r * (480 * size + 1):][:480 * size].view(dtype) for r in range(4)])
    row = np.arange(480).astype(dtype)
    cases = [(odd, odd_values), (np.broadcast_to(row, (4, 480)), np.tile(row, (4, 1))),
             (np.arange(4 * 480).astype(dtype).reshape(4, 480)[::-1], np.arange(4 * 480).astype(dtype).reshape(4, 480)[::-1].copy())]
    for x, want in cases:
        a, pitch, _ = e._check_host_audio(x)
        assert a.flags.c_contiguous and pitch == 480
        assert np.array_equal(a.view(np.uint8), np.ascontiguousarray(want).view(np.uint8))


def test_host_audio_check_refuses_other_dtypes_and_shapes():
    from microwakeword_b200.engine import MultiModelEngine, StreamEngine
    for cls in (StreamEngine, MultiModelEngine):
        e = _engine(cls)
        for bad in (np.zeros((4, 480), np.float64), np.zeros((4, 480), np.float16), np.zeros((4, 480), np.int32),
                    np.zeros((3, 480), np.float32), np.zeros((4, 480, 1), np.float32), np.zeros(480, np.float32),
                    [[0.0] * 480] * 4):
            with pytest.raises(ValueError):
                e._check_host_audio(bad)


def test_remote_dtype_selects_the_entry_point():
    import torch
    from microwakeword_b200.engine import MultiModelEngine, StreamEngine
    for cls, name in ((StreamEngine, "mww_predict_clip_remote"), (MultiModelEngine, "mww_predict_clip_remote_multi")):
        e = _engine(cls)
        L = e._L
        for dt in (np.int16, "int16", torch.int16):
            assert e._remote_fn(dt, name) is getattr(L, name)
        for dt in (np.float32, "float32", torch.float32):
            assert e._remote_fn(dt, name) is getattr(L, name + "_f32")
        for dt in (np.float64, np.uint16, torch.float64, torch.bfloat16, "pcm"):
            with pytest.raises(ValueError):
                e._remote_fn(dt, name)
        with pytest.raises(ValueError):                       # refused before any device work
            e.predict_clip_remote(0, 480, dtype=np.float64)
