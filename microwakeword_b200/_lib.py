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
MWW_RATE_PER_STREAM = 0
MWW_G711_ULAW, MWW_G711_ALAW = 1, 2
MWW_FORMAT_S16, MWW_FORMAT_ULAW, MWW_FORMAT_ALAW, MWW_FORMAT_F32 = 0, 1, 2, 3

# every symbol include/mww.h declares (checked by tests/test_capi_symbols.py)
EXPORTS = (
    "mww_create", "mww_destroy", "mww_last_error", "mww_get_info", "mww_reset", "mww_reset_frontend",
    "mww_features", "mww_infer_features", "mww_predict_clip", "mww_predict_clip_host",
    "mww_get_state", "mww_set_state", "mww_launch_count", "mww_profile_enable", "mww_profile_read", "mww_timeline_read",
    "mww_moving_average", "mww_false_accept_counts", "mww_positive_scores", "mww_copy_async",
    "mww_ipc_alloc", "mww_ipc_open", "mww_ipc_close", "mww_ipc_free",
    "mww_predict_clip_remote", "mww_reset_device_ids", "mww_host_alloc", "mww_host_alloc_wc", "mww_host_free", "mww_bind_host_thread",
    "mww_set_window_step", "mww_features_f32", "mww_predict_clip_f32", "mww_copy_nn_state", "mww_accuracy_counts",
    "mww_create_multi", "mww_model_count", "mww_get_model_info", "mww_predict_clip_multi", "mww_predict_clip_multi_f32",
    "mww_predict_clip_host_multi", "mww_predict_clip_remote_multi", "mww_get_model_state", "mww_set_model_state",
    "mww_predict_clip_host_f32", "mww_predict_clip_host_multi_f32", "mww_predict_clip_remote_f32", "mww_predict_clip_remote_multi_f32",
    "mww_create_multi_streams", "mww_set_model_streams", "mww_get_model_streams",
    "mww_stream_layout_get", "mww_export_streams", "mww_import_streams",
    "mww_set_input_rate", "mww_get_input_rate", "mww_get_resampler_state", "mww_set_resampler_state", "mww_resample_taps",
    "mww_set_stream_rates", "mww_get_stream_rates", "mww_rate_inputs",
    "mww_set_stream_formats", "mww_get_stream_formats", "mww_features_mixed", "mww_predict_clip_mixed", "mww_predict_clip_multi_mixed",
    "mww_predict_clip_host_mixed", "mww_predict_clip_host_multi_mixed", "mww_predict_clip_remote_mixed",
    "mww_predict_clip_remote_multi_mixed",
    "mww_detector_create", "mww_detector_destroy", "mww_detector_update", "mww_detector_drain", "mww_detector_buffers",
    "mww_detector_reset", "mww_detector_reset_device", "mww_detector_get_state", "mww_detector_set_state",
    "mww_multi_detector_create", "mww_multi_detector_update", "mww_multi_detector_get_state", "mww_multi_detector_set_state",
    "mww_set_detector_cutoffs", "mww_get_detector_cutoffs", "mww_set_multi_detector_cutoffs", "mww_get_multi_detector_cutoffs",
    "mww_features_g711", "mww_predict_clip_g711", "mww_predict_clip_host_g711", "mww_predict_clip_remote_g711",
    "mww_predict_clip_multi_g711", "mww_predict_clip_host_multi_g711", "mww_predict_clip_remote_multi_g711",
    "mww_set_audio_history", "mww_get_audio_history", "mww_read_audio_history", "mww_read_audio_history_device_ids",
    "mww_get_detector_layout", "mww_export_detector_rows", "mww_import_detector_rows",
    "mww_verifier_create", "mww_verifier_destroy", "mww_verifier_info", "mww_verify_streams", "mww_verify_detections",
    "mww_endpointer_create", "mww_endpointer_destroy", "mww_endpointer_info", "mww_endpointer_update", "mww_endpointer_arm",
    "mww_endpointer_arm_device", "mww_endpointer_disarm", "mww_endpointer_reset", "mww_endpointer_reset_device",
    "mww_endpointer_drain", "mww_endpointer_buffers", "mww_endpointer_get_state", "mww_endpointer_set_state",
    "mww_endpointer_read_commands",
    "mww_write_audio_history", "mww_get_endpointer_layout", "mww_export_endpointer_rows", "mww_import_endpointer_rows",
    "mww_get_resampler_layout", "mww_export_resampled_streams", "mww_import_resampled_streams",
    "mww_time_detector_events", "mww_update_detector_at", "mww_update_multi_detector_at", "mww_get_detector_positions",
    "mww_drain_detector_at", "mww_read_audio_history_at", "mww_verify_detections_at",
    "mww_group_detector_events", "mww_set_detector_groups", "mww_get_detector_groups", "mww_set_multi_detector_groups",
    "mww_get_multi_detector_groups", "mww_flush_detector_groups", "mww_drain_detector_groups", "mww_get_detector_group_windows",
    "mww_set_detector_group_windows",
    "mww_media_guard_create", "mww_media_guard_destroy", "mww_media_guard_info", "mww_media_check_streams",
    "mww_media_check_detections_at", "mww_media_register", "mww_media_clear_registered", "mww_media_clear_ring",
    "mww_media_get_state", "mww_media_set_state",
    "mww_playback_guard_create", "mww_playback_guard_destroy", "mww_playback_guard_info", "mww_playback_write", "mww_playback_read",
    "mww_playback_reset", "mww_playback_get_heads", "mww_playback_check_streams", "mww_playback_check_detections_at",
    "mww_arbitrate_detector_groups", "mww_drain_detector_arbitrated", "mww_get_detector_group_levels", "mww_set_detector_group_levels",
    "mww_endpointer_arm_at", "mww_endpointer_arm_at_device", "mww_endpointer_get_mutes", "mww_endpointer_set_mutes",
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


class MwwStreamLayout(ctypes.Structure):
    """mww_stream_layout of include/mww.h: what travels beside exported stream records"""
    _fields_ = [
        ("record_bytes", ctypes.c_int64), ("n_models", ctypes.c_int32), ("frontend_buffered", ctypes.c_int32),
        ("hop_samples", ctypes.c_int32), ("pending_rows", ctypes.c_int32 * 64), ("model_hash", ctypes.c_uint64 * 64),
        ("rows_are_features", ctypes.c_uint8 * 64),
    ]


class MwwResamplerLayout(ctypes.Structure):
    """mww_resampler_layout of include/mww.h: what travels beside resampled stream records, with the streams' rates"""
    _fields_ = [
        ("record_bytes", ctypes.c_int64), ("resampler_off", ctypes.c_int64), ("rate", ctypes.c_int32), ("reserved", ctypes.c_int32),
        ("inputs_seen", ctypes.c_int64), ("samples16_seen", ctypes.c_int64),
    ]


class MwwEvent(ctypes.Structure):
    """mww_event of include/mww.h: one detection of a streaming detector"""
    _fields_ = [("stream", ctypes.c_int32), ("reserved", ctypes.c_int32), ("step", ctypes.c_int64), ("score", ctypes.c_float),
                ("pad", ctypes.c_int32)]


MWW_DETECT_OFF, MWW_DETECT_WAKE, MWW_DETECT_VAD = 0, 1, 2


class MwwDetectRule(ctypes.Structure):
    """mww_detect_rule of include/mww.h: one model's rule in a models detector"""
    _fields_ = [("role", ctypes.c_int32), ("window", ctypes.c_int32), ("cooldown_slices", ctypes.c_int32), ("pad", ctypes.c_int32),
                ("cutoff", ctypes.c_double)]


class MwwDetectorLayout(ctypes.Structure):
    """mww_detector_layout of include/mww.h: what travels beside exported detector records"""
    _fields_ = [
        ("record_bytes", ctypes.c_int64), ("multi", ctypes.c_int32), ("n_models", ctypes.c_int32),
        ("role", ctypes.c_int32 * 64), ("window", ctypes.c_int32 * 64), ("cooldown_slices", ctypes.c_int32 * 64),
    ]


class MwwVerifyRule(ctypes.Structure):
    """mww_verify_rule of include/mww.h: what a verifier reads, and how it scores and confirms"""
    _fields_ = [("n_samples", ctypes.c_int32), ("window", ctypes.c_int32), ("ignore_steps", ctypes.c_int32), ("pad", ctypes.c_int32),
                ("cutoff", ctypes.c_double)]


class MwwVerifierDesc(ctypes.Structure):
    """mww_verifier_desc of include/mww.h (mww_verifier_info)"""
    _fields_ = [("slots", ctypes.c_int32), ("steps", ctypes.c_int32), ("device", ctypes.c_int32), ("pad", ctypes.c_int32),
                ("rule", MwwVerifyRule), ("launches", ctypes.c_int64)]


class MwwMediaRule(ctypes.Structure):
    """mww_media_rule of include/mww.h: what a media guard hears and when two fingerprints match"""
    _fields_ = [("n_samples", ctypes.c_int32), ("max_lag", ctypes.c_int32), ("min_overlap", ctypes.c_int32), ("max_ber_milli", ctypes.c_int32),
                ("min_matches", ctypes.c_int32), ("ring", ctypes.c_int32), ("max_media", ctypes.c_int32), ("max_media_samples", ctypes.c_int32),
                ("window_samples", ctypes.c_int64)]


class MwwMediaGuardDesc(ctypes.Structure):
    """mww_media_guard_desc of include/mww.h (mww_media_guard_info)"""
    _fields_ = [("slots", ctypes.c_int32), ("frames", ctypes.c_int32), ("device", ctypes.c_int32), ("n_media", ctypes.c_int32),
                ("rule", MwwMediaRule), ("ring_fill", ctypes.c_int64), ("ring_count", ctypes.c_int64), ("launches", ctypes.c_int64)]


class MwwPlaybackRule(ctypes.Structure):
    """mww_playback_rule of include/mww.h: the reference clip a playback guard scores, and its cutoff"""
    _fields_ = [("n_samples", ctypes.c_int32), ("window", ctypes.c_int32), ("ignore_steps", ctypes.c_int32), ("pad", ctypes.c_int32),
                ("min_delay", ctypes.c_int64), ("max_delay", ctypes.c_int64), ("cutoff", ctypes.c_double)]


class MwwPlaybackGuardDesc(ctypes.Structure):
    """mww_playback_guard_desc of include/mww.h (mww_playback_guard_info)"""
    _fields_ = [("slots", ctypes.c_int32), ("steps", ctypes.c_int32), ("rows", ctypes.c_int32), ("rows_used", ctypes.c_int32),
                ("capacity", ctypes.c_int32), ("l_ref", ctypes.c_int32), ("device", ctypes.c_int32), ("pad", ctypes.c_int32),
                ("rule", MwwPlaybackRule), ("launches", ctypes.c_int64)]


MWW_ENDPOINT_END_OF_SPEECH, MWW_ENDPOINT_NO_SPEECH, MWW_ENDPOINT_MAX_LENGTH = 1, 2, 3


class MwwEndpointRule(ctypes.Structure):
    """mww_endpoint_rule of include/mww.h: an endpointer's VAD rule and segmenter limits, in model steps"""
    _fields_ = [("vad_window", ctypes.c_int32), ("speech_steps", ctypes.c_int32), ("silence_steps", ctypes.c_int32),
                ("timeout_steps", ctypes.c_int32), ("max_steps", ctypes.c_int32), ("lookback_steps", ctypes.c_int32),
                ("vad_cutoff", ctypes.c_double)]


class MwwEndpointEvent(ctypes.Structure):
    """mww_endpoint_event of include/mww.h: one command that ended"""
    _fields_ = [("stream", ctypes.c_int32), ("reason", ctypes.c_int32), ("start_sample", ctypes.c_int64), ("end_sample", ctypes.c_int64),
                ("speech_end_sample", ctypes.c_int64), ("steps", ctypes.c_int32), ("pad", ctypes.c_int32)]


class MwwEndpointerDesc(ctypes.Structure):
    """mww_endpointer_desc of include/mww.h (mww_endpointer_info)"""
    _fields_ = [("n_rows", ctypes.c_int32), ("model", ctypes.c_int32), ("stride", ctypes.c_int32), ("hop_samples", ctypes.c_int32),
                ("capacity", ctypes.c_int32), ("device", ctypes.c_int32), ("rule", MwwEndpointRule), ("steps", ctypes.c_int64),
                ("launches", ctypes.c_int64)]


class MwwEndpointState(ctypes.Structure):
    """mww_endpoint_state of include/mww.h (mww_endpointer_get_state / _set_state): host pointers to the row arrays, the
    baseline counters, the steps consumed and the last 64 step positions"""
    _fields_ = [("hist", ctypes.c_void_p), ("seen", ctypes.c_void_p), ("flags", ctypes.c_void_p), ("armed", ctypes.c_void_p),
                ("elapsed", ctypes.c_void_p), ("run", ctypes.c_void_p), ("silence", ctypes.c_void_p), ("heard", ctypes.c_void_p),
                ("start_sample", ctypes.c_void_p), ("speech_end_sample", ctypes.c_void_p), ("samples_seen", ctypes.c_int64),
                ("buffered", ctypes.c_int64), ("pending", ctypes.c_int64), ("steps", ctypes.c_int64), ("positions", ctypes.c_int64 * 64)]


class MwwEndpointerLayout(ctypes.Structure):
    """mww_endpointer_layout of include/mww.h: what travels beside exported endpointer records"""
    _fields_ = [("record_bytes", ctypes.c_int64), ("vad_window", ctypes.c_int32), ("stride", ctypes.c_int32),
                ("hop_samples", ctypes.c_int32), ("buffered", ctypes.c_int32), ("pending", ctypes.c_int32), ("pad", ctypes.c_int32),
                ("samples_seen", ctypes.c_int64), ("steps", ctypes.c_int64)]


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
    for name in ("mww_predict_clip_host", "mww_predict_clip_host_f32"):
        getattr(L, name).restype = i32
        getattr(L, name).argtypes = [vp, vp, i32, ll, vp, i32, pi]
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
    L.mww_accuracy_counts.restype = i32
    L.mww_accuracy_counts.argtypes = [vp, vp, vp, i32, i32, vp, vp, vp]
    L.mww_copy_nn_state.restype = i32
    L.mww_copy_nn_state.argtypes = [vp, vp, vp, vp, i32, vp]
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
    for name in ("mww_predict_clip_remote", "mww_predict_clip_remote_f32"):
        getattr(L, name).restype = i32
        getattr(L, name).argtypes = [vp, vp, i32, ll, vp, i32, pi, i32, vp]
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
    L.mww_create_multi.restype = i32
    L.mww_create_multi.argtypes = [vp, vp, i32, i32, i32, ctypes.POINTER(vp)]
    L.mww_model_count.restype = i32
    L.mww_model_count.argtypes = [vp]
    L.mww_get_model_info.restype = i32
    L.mww_get_model_info.argtypes = [vp, i32, ctypes.POINTER(MwwInfo)]
    for name in ("mww_predict_clip_multi", "mww_predict_clip_multi_f32"):
        getattr(L, name).restype = i32
        getattr(L, name).argtypes = [vp, vp, i32, ll, vp, vp, vp, vp]
    for name in ("mww_predict_clip_host_multi", "mww_predict_clip_host_multi_f32"):
        getattr(L, name).restype = i32
        getattr(L, name).argtypes = [vp, vp, i32, ll, vp, vp, vp]
    for name in ("mww_predict_clip_remote_multi", "mww_predict_clip_remote_multi_f32"):
        getattr(L, name).restype = i32
        getattr(L, name).argtypes = [vp, vp, i32, ll, vp, vp, vp, i32, vp]
    L.mww_get_model_state.restype = i32
    L.mww_get_model_state.argtypes = [vp, i32, vp, vp]
    L.mww_set_model_state.restype = i32
    L.mww_set_model_state.argtypes = [vp, i32, vp, vp, i32]
    L.mww_create_multi_streams.restype = i32
    L.mww_create_multi_streams.argtypes = [vp, vp, i32, i32, i32, vp, vp, ctypes.POINTER(vp)]
    L.mww_set_model_streams.restype = i32
    L.mww_set_model_streams.argtypes = [vp, i32, vp, i32, vp]
    L.mww_get_model_streams.restype = i32
    L.mww_get_model_streams.argtypes = [vp, i32, vp, i32, pi]
    L.mww_stream_layout_get.restype = i32
    L.mww_stream_layout_get.argtypes = [vp, ctypes.POINTER(MwwStreamLayout)]
    L.mww_export_streams.restype = i32
    L.mww_export_streams.argtypes = [vp, vp, i32, vp, ctypes.POINTER(MwwStreamLayout), vp]
    L.mww_import_streams.restype = i32
    L.mww_import_streams.argtypes = [vp, vp, i32, vp, ctypes.POINTER(MwwStreamLayout), vp]
    L.mww_get_resampler_layout.restype = i32
    L.mww_get_resampler_layout.argtypes = [vp, ctypes.POINTER(MwwResamplerLayout)]
    L.mww_export_resampled_streams.restype = i32
    L.mww_export_resampled_streams.argtypes = [vp, vp, i32, vp, ctypes.POINTER(MwwStreamLayout), ctypes.POINTER(MwwResamplerLayout), vp, vp]
    L.mww_import_resampled_streams.restype = i32
    L.mww_import_resampled_streams.argtypes = [vp, vp, i32, vp, ctypes.POINTER(MwwStreamLayout), ctypes.POINTER(MwwResamplerLayout), vp, vp]
    L.mww_set_input_rate.restype = i32
    L.mww_set_input_rate.argtypes = [vp, i32]
    L.mww_get_input_rate.restype = i32
    L.mww_get_input_rate.argtypes = [vp, pi, ctypes.POINTER(ll)]
    L.mww_get_resampler_state.restype = i32
    L.mww_get_resampler_state.argtypes = [vp, vp, ctypes.POINTER(ll)]
    L.mww_set_resampler_state.restype = i32
    L.mww_set_resampler_state.argtypes = [vp, vp, ll]
    L.mww_resample_taps.restype = i32
    L.mww_resample_taps.argtypes = [i32, vp, i32, pi, pi, pi]
    L.mww_set_stream_rates.restype = i32
    L.mww_set_stream_rates.argtypes = [vp, vp, vp, i32, vp]
    L.mww_get_stream_rates.restype = i32
    L.mww_get_stream_rates.argtypes = [vp, vp, ctypes.POINTER(ll)]
    L.mww_rate_inputs.restype = i32
    L.mww_rate_inputs.argtypes = [i32, ll, ctypes.POINTER(ll)]
    L.mww_detector_create.restype = i32
    L.mww_detector_create.argtypes = [i32, i32, i32, ctypes.c_double, i32, i32, vp, ctypes.POINTER(vp)]
    L.mww_detector_destroy.restype = i32
    L.mww_detector_destroy.argtypes = [vp]
    L.mww_detector_update.restype = i32
    L.mww_detector_update.argtypes = [vp, vp, i32, ll, vp]
    L.mww_detector_drain.restype = i32
    L.mww_detector_drain.argtypes = [vp, vp, i32, ctypes.POINTER(ll), vp]
    L.mww_detector_buffers.restype = i32
    L.mww_detector_buffers.argtypes = [vp, ctypes.POINTER(vp), ctypes.POINTER(vp), ctypes.POINTER(vp), pi]
    for name in ("mww_detector_reset", "mww_detector_reset_device"):
        getattr(L, name).restype = i32
        getattr(L, name).argtypes = [vp, vp, i32, vp]
    for name in ("mww_detector_get_state", "mww_detector_set_state"):
        getattr(L, name).restype = i32
        getattr(L, name).argtypes = [vp, vp, vp, vp]
    L.mww_multi_detector_create.restype = i32
    L.mww_multi_detector_create.argtypes = [vp, ctypes.POINTER(MwwDetectRule), i32, ctypes.POINTER(vp)]
    L.mww_multi_detector_update.restype = i32
    L.mww_multi_detector_update.argtypes = [vp, vp, vp, vp, vp, vp]
    for name in ("mww_multi_detector_get_state", "mww_multi_detector_set_state"):
        getattr(L, name).restype = i32
        getattr(L, name).argtypes = [vp, i32, vp, vp, vp]
    L.mww_set_detector_cutoffs.restype = i32
    L.mww_set_detector_cutoffs.argtypes = [vp, vp, vp, i32, vp]
    L.mww_get_detector_cutoffs.restype = i32
    L.mww_get_detector_cutoffs.argtypes = [vp, vp]
    L.mww_set_multi_detector_cutoffs.restype = i32
    L.mww_set_multi_detector_cutoffs.argtypes = [vp, i32, vp, vp, i32, vp]
    L.mww_get_multi_detector_cutoffs.restype = i32
    L.mww_get_multi_detector_cutoffs.argtypes = [vp, i32, vp]
    # G.711 forms: the int16 counterpart's arguments with the law (MWW_G711_*) after the audio pointer
    for name in ("mww_features", "mww_predict_clip", "mww_predict_clip_host", "mww_predict_clip_remote", "mww_predict_clip_multi",
                 "mww_predict_clip_host_multi", "mww_predict_clip_remote_multi"):
        args = getattr(L, name).argtypes
        getattr(L, name + "_g711").restype = i32
        getattr(L, name + "_g711").argtypes = args[:2] + [i32] + args[2:]
        # mixed rows (a format per stream): the int16 counterpart's arguments, the audio as bytes with a stride in bytes
        getattr(L, name + "_mixed").restype = i32
        getattr(L, name + "_mixed").argtypes = list(args)
    L.mww_set_stream_formats.restype = i32
    L.mww_set_stream_formats.argtypes = [vp, vp, vp, i32, vp]
    L.mww_get_stream_formats.restype = i32
    L.mww_get_stream_formats.argtypes = [vp, vp]
    L.mww_set_audio_history.restype = i32
    L.mww_set_audio_history.argtypes = [vp, i32, vp]
    L.mww_get_audio_history.restype = i32
    L.mww_get_audio_history.argtypes = [vp, pi, ctypes.POINTER(ll)]
    for name in ("mww_read_audio_history", "mww_read_audio_history_device_ids"):
        getattr(L, name).restype = i32
        getattr(L, name).argtypes = [vp, vp, i32, i32, vp, ll, vp]
    L.mww_get_detector_layout.restype = i32
    L.mww_get_detector_layout.argtypes = [vp, ctypes.POINTER(MwwDetectorLayout)]
    for name in ("mww_export_detector_rows", "mww_import_detector_rows"):
        getattr(L, name).restype = i32
        getattr(L, name).argtypes = [vp, vp, i32, vp, ctypes.POINTER(MwwDetectorLayout), vp]
    L.mww_verifier_create.restype = i32
    L.mww_verifier_create.argtypes = [vp, sz, i32, i32, ctypes.POINTER(MwwVerifyRule), ctypes.POINTER(vp)]
    L.mww_verifier_destroy.restype = i32
    L.mww_verifier_destroy.argtypes = [vp]
    L.mww_verifier_info.restype = i32
    L.mww_verifier_info.argtypes = [vp, ctypes.POINTER(MwwVerifierDesc)]
    L.mww_verify_streams.restype = i32
    L.mww_verify_streams.argtypes = [vp, vp, vp, i32, vp, vp, vp]
    L.mww_verify_detections.restype = i32
    L.mww_verify_detections.argtypes = [vp, vp, vp, i32, vp, vp, vp]
    L.mww_endpointer_create.restype = i32
    L.mww_endpointer_create.argtypes = [vp, i32, ctypes.POINTER(MwwEndpointRule), i32, ctypes.POINTER(vp)]
    L.mww_endpointer_destroy.restype = i32
    L.mww_endpointer_destroy.argtypes = [vp]
    L.mww_endpointer_info.restype = i32
    L.mww_endpointer_info.argtypes = [vp, ctypes.POINTER(MwwEndpointerDesc)]
    L.mww_endpointer_update.restype = i32
    L.mww_endpointer_update.argtypes = [vp, vp, i32, ll, vp]
    for name in ("mww_endpointer_arm", "mww_endpointer_arm_device", "mww_endpointer_disarm", "mww_endpointer_reset",
                 "mww_endpointer_reset_device"):
        getattr(L, name).restype = i32
        getattr(L, name).argtypes = [vp, vp, i32, vp]
    L.mww_endpointer_drain.restype = i32
    L.mww_endpointer_drain.argtypes = [vp, vp, i32, ctypes.POINTER(ll), vp]
    L.mww_endpointer_buffers.restype = i32
    L.mww_endpointer_buffers.argtypes = [vp, ctypes.POINTER(vp), ctypes.POINTER(vp), ctypes.POINTER(vp), ctypes.POINTER(vp), pi]
    L.mww_endpointer_get_state.restype = i32
    L.mww_endpointer_get_state.argtypes = [vp, ctypes.POINTER(MwwEndpointState)]
    L.mww_endpointer_set_state.restype = i32
    L.mww_endpointer_set_state.argtypes = [vp, ctypes.POINTER(MwwEndpointState)]
    L.mww_endpointer_read_commands.restype = i32
    L.mww_endpointer_read_commands.argtypes = [vp, vp, ll, ll, i32, vp, ll, vp, vp]
    L.mww_write_audio_history.restype = i32
    L.mww_write_audio_history.argtypes = [vp, vp, i32, i32, vp, ll, vp]
    L.mww_get_endpointer_layout.restype = i32
    L.mww_get_endpointer_layout.argtypes = [vp, ctypes.POINTER(MwwEndpointerLayout)]
    for name in ("mww_export_endpointer_rows", "mww_import_endpointer_rows"):
        getattr(L, name).restype = i32
        getattr(L, name).argtypes = [vp, vp, i32, vp, ctypes.POINTER(MwwEndpointerLayout), vp]
    for name in ("mww_endpointer_arm_at", "mww_endpointer_arm_at_device"):
        getattr(L, name).restype = i32
        getattr(L, name).argtypes = [vp, vp, vp, i32, ll, vp]
    for name in ("mww_endpointer_get_mutes", "mww_endpointer_set_mutes"):
        getattr(L, name).restype = i32
        getattr(L, name).argtypes = [vp, vp]
    L.mww_time_detector_events.restype = i32
    L.mww_time_detector_events.argtypes = [vp]
    L.mww_update_detector_at.restype = i32
    L.mww_update_detector_at.argtypes = [vp, vp, i32, ll, ll, ll, vp]
    L.mww_update_multi_detector_at.restype = i32
    L.mww_update_multi_detector_at.argtypes = [vp, vp, vp, vp, vp, vp, ll, vp]
    L.mww_get_detector_positions.restype = i32
    L.mww_get_detector_positions.argtypes = [vp, ctypes.POINTER(vp)]
    L.mww_drain_detector_at.restype = i32
    L.mww_drain_detector_at.argtypes = [vp, vp, vp, i32, ctypes.POINTER(ll), vp]
    L.mww_read_audio_history_at.restype = i32
    L.mww_read_audio_history_at.argtypes = [vp, vp, vp, i32, i32, vp, ll, vp]
    L.mww_verify_detections_at.restype = i32
    L.mww_verify_detections_at.argtypes = [vp, vp, vp, i32, ll, vp, vp, vp]
    L.mww_group_detector_events.restype = i32
    L.mww_group_detector_events.argtypes = [vp, i32, ll]
    for name in ("mww_set_detector_groups", "mww_set_multi_detector_groups"):
        getattr(L, name).restype = i32
        getattr(L, name).argtypes = [vp, vp, vp, i32, vp]
    for name in ("mww_get_detector_groups", "mww_get_multi_detector_groups", "mww_get_detector_group_windows", "mww_set_detector_group_windows"):
        getattr(L, name).restype = i32
        getattr(L, name).argtypes = [vp, vp]
    L.mww_flush_detector_groups.restype = i32
    L.mww_flush_detector_groups.argtypes = [vp, vp]
    L.mww_drain_detector_groups.restype = i32
    L.mww_drain_detector_groups.argtypes = [vp, vp, vp, vp, vp, i32, ctypes.POINTER(ll), vp]
    L.mww_media_guard_create.restype = i32
    L.mww_media_guard_create.argtypes = [i32, i32, ctypes.POINTER(MwwMediaRule), ctypes.POINTER(vp)]
    L.mww_media_guard_destroy.restype = i32
    L.mww_media_guard_destroy.argtypes = [vp]
    L.mww_media_guard_info.restype = i32
    L.mww_media_guard_info.argtypes = [vp, ctypes.POINTER(MwwMediaGuardDesc)]
    L.mww_media_check_streams.restype = i32
    L.mww_media_check_streams.argtypes = [vp, vp, vp, vp, vp, i32, vp, vp, vp, vp, vp]
    L.mww_media_check_detections_at.restype = i32
    L.mww_media_check_detections_at.argtypes = [vp, vp, vp, i32, ll, vp, vp, vp, vp, vp]
    L.mww_media_register.restype = i32
    L.mww_media_register.argtypes = [vp, vp, i32, pi, vp]
    for name in ("mww_media_clear_registered", "mww_media_clear_ring"):
        getattr(L, name).restype = i32
        getattr(L, name).argtypes = [vp]
    L.mww_media_get_state.restype = i32
    L.mww_media_get_state.argtypes = [vp, vp, ctypes.POINTER(ll)]
    L.mww_media_set_state.restype = i32
    L.mww_media_set_state.argtypes = [vp, vp, ll]
    L.mww_playback_guard_create.restype = i32
    L.mww_playback_guard_create.argtypes = [vp, vp, sz, i32, i32, i32, ctypes.POINTER(MwwPlaybackRule), ctypes.POINTER(vp)]
    L.mww_playback_guard_destroy.restype = i32
    L.mww_playback_guard_destroy.argtypes = [vp]
    L.mww_playback_guard_info.restype = i32
    L.mww_playback_guard_info.argtypes = [vp, ctypes.POINTER(MwwPlaybackGuardDesc)]
    L.mww_playback_write.restype = i32
    L.mww_playback_write.argtypes = [vp, vp, vp, i32, vp, i32, ll, vp]
    L.mww_playback_read.restype = i32
    L.mww_playback_read.argtypes = [vp, vp, vp, i32, i32, vp, ll, vp]
    L.mww_playback_reset.restype = i32
    L.mww_playback_reset.argtypes = [vp, vp, i32, vp]
    L.mww_playback_get_heads.restype = i32
    L.mww_playback_get_heads.argtypes = [vp, vp, vp]
    L.mww_playback_check_streams.restype = i32
    L.mww_playback_check_streams.argtypes = [vp, vp, vp, i32, vp, vp, vp, vp, vp]
    L.mww_playback_check_detections_at.restype = i32
    L.mww_playback_check_detections_at.argtypes = [vp, vp, i32, ll, vp, vp, vp, vp, vp]
    L.mww_arbitrate_detector_groups.restype = i32
    L.mww_arbitrate_detector_groups.argtypes = [vp, vp, i32, i32]
    L.mww_drain_detector_arbitrated.restype = i32
    L.mww_drain_detector_arbitrated.argtypes = [vp, vp, vp, vp, vp, vp, i32, ctypes.POINTER(ll), vp]
    for name in ("mww_get_detector_group_levels", "mww_set_detector_group_levels"):
        getattr(L, name).restype = i32
        getattr(L, name).argtypes = [vp, vp]
    _lib = L
    return L


def check(handle, rc: int) -> None:
    if rc != 0:
        msg = lib().mww_last_error(handle)
        raise MwwError(rc, msg.decode() if msg else "unknown error")
