"""ctypes binding of libmww_b200.so (C-ABI declared in include/mww.h).

There is deliberately no CPU fallback: if the shared library is missing it is built with nvcc, and
if that is impossible -- or no CUDA device is present at `mww_create` time -- the caller gets an
exception, never a silently different code path.
"""

from __future__ import annotations

import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.path.join(_HERE, "libmww_b200.so")

MWW_ROWS_U16, MWW_ROWS_F32, MWW_ROWS_I8 = 0, 1, 2

# every symbol include/mww.h declares (checked by tests/test_capi_symbols.py)
EXPORTS = (
    "mww_create", "mww_destroy", "mww_last_error", "mww_get_info", "mww_reset", "mww_reset_frontend",
    "mww_features", "mww_infer_features", "mww_predict_clip", "mww_predict_clip_host",
    "mww_get_state", "mww_set_state", "mww_launch_count", "mww_profile_enable", "mww_profile_read", "mww_timeline_read",
    "mww_moving_average", "mww_false_accept_counts", "mww_positive_scores", "mww_copy_async",
    "mww_ipc_alloc", "mww_ipc_open", "mww_ipc_close", "mww_ipc_free",
    "mww_predict_clip_remote", "mww_reset_device_ids", "mww_host_alloc", "mww_host_alloc_wc", "mww_host_free", "mww_bind_host_thread",
    "mww_set_window_step", "mww_features_f32", "mww_predict_clip_f32",
)


class MwwInfo(ctypes.Structure):
    _fields_ = [
        ("n_streams", ctypes.c_int32), ("device", ctypes.c_int32), ("is_quantized", ctypes.c_int32),
        ("input_feature_slices", ctypes.c_int32), ("num_features", ctypes.c_int32),
        ("input_scale", ctypes.c_float), ("input_zero_point", ctypes.c_int32),
        ("output_scale", ctypes.c_float), ("output_zero_point", ctypes.c_int32),
        ("state_bytes_per_stream", ctypes.c_int32), ("frontend_buffered", ctypes.c_int32),
        ("pending_rows", ctypes.c_int32), ("sm_count", ctypes.c_int32), ("macs_per_step", ctypes.c_int32),
        ("hop_samples", ctypes.c_int32),
    ]


class MwwError(RuntimeError):
    def __init__(self, code: int, message: str):
        super().__init__("libmww_b200 error %d: %s" % (code, message))
        self.code = code


_lib = None


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    from . import build as _build
    if not os.path.exists(SO_PATH):
        _build.build()                 # raises if nvcc is unavailable
    elif os.path.exists(_build.NVCC) and _build._stale():
        _build.build()                 # sources newer than the binary: never load a library with an older ABI
    L = ctypes.CDLL(SO_PATH)
    vp, i32, ll, sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_size_t
    pi = ctypes.POINTER(ctypes.c_int)
    L.mww_create.restype = i32
    L.mww_create.argtypes = [vp, sz, i32, i32, ctypes.POINTER(vp)]
    L.mww_destroy.restype = i32
    L.mww_destroy.argtypes = [vp]
    L.mww_last_error.restype = ctypes.c_char_p
    L.mww_last_error.argtypes = [vp]
    L.mww_get_info.restype = i32
    L.mww_get_info.argtypes = [vp, ctypes.POINTER(MwwInfo)]
    L.mww_reset.restype = i32
    L.mww_reset.argtypes = [vp, vp, i32, vp]
    L.mww_reset_frontend.restype = i32
    L.mww_reset_frontend.argtypes = [vp, vp]
    L.mww_features.restype = i32
    L.mww_features.argtypes = [vp, vp, i32, ll, vp, i32, pi, vp]
    L.mww_infer_features.restype = i32
    L.mww_infer_features.argtypes = [vp, vp, i32, i32, ll, vp, i32, pi, vp]
    L.mww_predict_clip.restype = i32
    L.mww_predict_clip.argtypes = [vp, vp, i32, ll, vp, i32, pi, vp]
    L.mww_features_f32.restype = i32
    L.mww_features_f32.argtypes = [vp, vp, i32, ll, vp, i32, pi, vp]
    L.mww_predict_clip_f32.restype = i32
    L.mww_predict_clip_f32.argtypes = [vp, vp, i32, ll, vp, i32, pi, vp]
    L.mww_predict_clip_host.restype = i32
    L.mww_predict_clip_host.argtypes = [vp, vp, i32, ll, vp, i32, pi]
    L.mww_get_state.restype = i32
    L.mww_get_state.argtypes = [vp, vp, vp, vp, vp]
    L.mww_set_state.restype = i32
    L.mww_set_state.argtypes = [vp, vp, i32, vp, vp, vp, i32]
    L.mww_profile_enable.restype = i32
    L.mww_profile_enable.argtypes = [vp, i32]
    L.mww_profile_read.restype = i32
    L.mww_profile_read.argtypes = [vp, ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_longlong)]
    L.mww_timeline_read.restype = i32
    L.mww_timeline_read.argtypes = [vp, ctypes.POINTER(ctypes.c_float), i32, ctypes.POINTER(i32)]
    L.mww_moving_average.restype = i32
    L.mww_moving_average.argtypes = [vp, vp, vp, i32, i32, i32, vp, vp, vp]
    L.mww_false_accept_counts.restype = i32
    L.mww_false_accept_counts.argtypes = [vp, vp, vp, i32, i32, vp, i32, i32, vp, vp]
    L.mww_positive_scores.restype = i32
    L.mww_positive_scores.argtypes = [vp, vp, vp, i32, i32, i32, vp, vp]
    L.mww_launch_count.restype = ll
    L.mww_launch_count.argtypes = [vp]
    L.mww_copy_async.restype = i32
    L.mww_copy_async.argtypes = [vp, vp, sz, vp]
    L.mww_ipc_alloc.restype = i32
    L.mww_ipc_alloc.argtypes = [sz, i32, ctypes.POINTER(vp), ctypes.c_char_p]
    L.mww_ipc_open.restype = i32
    L.mww_ipc_open.argtypes = [ctypes.c_char_p, i32, ctypes.POINTER(vp)]
    L.mww_ipc_close.restype = i32
    L.mww_ipc_close.argtypes = [vp, i32]
    L.mww_ipc_free.restype = i32
    L.mww_ipc_free.argtypes = [vp, i32]
    L.mww_predict_clip_remote.restype = i32
    L.mww_predict_clip_remote.argtypes = [vp, vp, i32, ll, vp, i32, pi, i32, vp]
    L.mww_reset_device_ids.restype = i32
    L.mww_reset_device_ids.argtypes = [vp, vp, i32, vp]
    L.mww_host_alloc.restype = i32
    L.mww_host_alloc.argtypes = [sz, i32, ctypes.POINTER(vp), pi]
    L.mww_host_alloc_wc.restype = i32
    L.mww_host_alloc_wc.argtypes = [sz, i32, ctypes.POINTER(vp), pi]
    L.mww_host_free.restype = i32
    L.mww_host_free.argtypes = [vp]
    L.mww_set_window_step.restype = i32
    L.mww_set_window_step.argtypes = [vp, i32]
    L.mww_bind_host_thread.restype = i32
    L.mww_bind_host_thread.argtypes = [i32, pi]
    _lib = L
    return L


def check(handle, rc: int) -> None:
    if rc != 0:
        msg = lib().mww_last_error(handle)
        raise MwwError(rc, msg.decode() if msg else "unknown error")
