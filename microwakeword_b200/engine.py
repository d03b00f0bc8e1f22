"""StreamEngine: many independent audio streams on one H100, behind the C-ABI of include/mww.h.

Host-side mirror of what the reference does one stream at a time:
  * frontend  ...... microwakeword/audio/audio_utils.py:50-64 (ProcessSamples loop)
  * model step ..... microwakeword/inference.py:109-123 (set_tensor / invoke / get_tensor)
batched over `n_streams` streams that advance in lockstep.  PyTorch tensors are used only as
device buffers (`.data_ptr()`) and for the current CUDA stream; all arithmetic is in
libmww_b200.so.
"""

from __future__ import annotations

import ctypes

import numpy as np

from . import _lib
from .model_file import NUM_FEATURES

HOP = 160
WINDOW = 480
STATE_ELEMENTS = 4176      # okay_nabu; other architectures: StreamEngine.state_elements


def _torch():
    import torch  # deferred: `import microwakeword_b200` must work without initialising CUDA
    return torch


class _PinnedBlock:
    """Owner of one mww_host_alloc allocation; numpy arrays built on it keep it alive through their .base chain."""

    def __init__(self, nbytes: int, device: int, write_combined: bool = False):
        L = _lib.lib()
        ptr, node = ctypes.c_void_p(), ctypes.c_int(-1)
        alloc = L.mww_host_alloc_wc if write_combined else L.mww_host_alloc
        _lib.check(None, alloc(max(int(nbytes), 1), int(device), ctypes.byref(ptr), ctypes.byref(node)))
        self.ptr, self.nbytes, self.numa_node = ptr.value, int(nbytes), node.value
        self.__array_interface__ = {"shape": (max(int(nbytes), 1),), "typestr": "|u1", "data": (self.ptr, False), "version": 3}

    def __del__(self):
        try:
            if self.ptr:
                _lib.lib().mww_host_free(ctypes.c_void_p(self.ptr))
                self.ptr = None
        except Exception:
            pass


def host_array(shape, dtype=np.int16, device: int = 0, write_combined: bool = False) -> np.ndarray:
    """Pinned, GPU-local (NUMA) host array; `.base.base.numa_node` tells where it landed (-1: topology unknown).
    write_combined: for input buffers the CPU only writes and the GPU only reads (mww_host_alloc_wc; CPU reads are very slow)."""
    dtype = np.dtype(dtype)
    n = int(np.prod(shape)) * dtype.itemsize
    block = _PinnedBlock(n, device, write_combined)
    return np.asarray(block)[:n].view(dtype).reshape(shape)


def bind_host_thread(device: int) -> int:
    """Move the calling thread (and the threads it starts later) to the CPUs of the GPU's NUMA node; returns the node or -1."""
    node = ctypes.c_int(-1)
    _lib.check(None, _lib.lib().mww_bind_host_thread(int(device), ctypes.byref(node)))
    return node.value


class StreamEngine:
    """`model`: path to (or bytes of) an MWW container or a streaming ``.tflite`` flatbuffer (recognised and converted by
    ``tflite_file``, inference.py:36-45), or None for a frontend-only engine."""

    def __init__(self, model, n_streams: int = 1, device: int = 0):
        if isinstance(model, (bytes, bytearray, memoryview)):
            blob = bytes(model)
        elif model is None:
            blob = None
        else:
            with open(model, "rb") as f:
                blob = f.read()
        if blob is not None:
            from . import tflite_file
            if tflite_file.is_tflite(blob):
                blob = tflite_file.container_from_tflite(blob)      # raises TfliteError for graphs outside the hot path
        self._L = _lib.lib()
        self._h = ctypes.c_void_p()
        self._blob = blob  # keep alive during create
        rc = self._L.mww_create(blob, len(blob) if blob else 0, int(device), int(n_streams), ctypes.byref(self._h))
        if rc != 0:
            msg = self._L.mww_last_error(None)
            raise _lib.MwwError(rc, msg.decode() if msg else "mww_create failed")
        self.n_streams = int(n_streams)
        self.device = int(device)
        self.info = self._info()
        self.is_quantized = bool(self.info.is_quantized)
        # geometry of the loaded model (mww_get_info): feature rows per model step, ring-state elements per stream
        self.stride = max(int(self.info.input_feature_slices), 1)
        self.state_elements = int(self.info.state_bytes_per_stream) // (1 if self.is_quantized else 4) if blob is not None else 0
        self.hop = HOP          # samples between feature windows (set_window_step)

    # ------------------------------------------------------------------ plumbing
    def close(self):
        if getattr(self, "_h", None):
            self._L.mww_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _info(self):
        info = _lib.MwwInfo()
        _lib.check(self._h, self._L.mww_get_info(self._h, ctypes.byref(info)))
        return info

    def _cu_stream(self):
        torch = _torch()
        return ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _dev(self):
        return _torch().device("cuda", self.device)

    @property
    def frontend_buffered(self) -> int:
        return self._info().frontend_buffered

    @property
    def pending_rows(self) -> int:
        return self._info().pending_rows

    @property
    def launch_count(self) -> int:
        return int(self._L.mww_launch_count(self._h))

    def _check_audio(self, audio):
        """-> (n_samples, row pitch in samples, is_float32).  float32 audio is converted to int16 inside the frontend kernels,
        exactly as audio_utils.to_int16 converts it on the host; other float dtypes are refused (float64 keeps its exact host
        conversion: rounding it to float32 first could move a sample across an integer boundary after the x 32768)."""
        torch = _torch()
        if (audio.dtype not in (torch.int16, torch.float32) or audio.dim() != 2 or audio.shape[0] != self.n_streams
                or not audio.is_cuda):
            raise ValueError("audio must be a CUDA int16 or float32 tensor of shape [n_streams=%d, n_samples]" % self.n_streams)
        if audio.stride(1) != 1 and audio.shape[1] > 1:
            raise ValueError("audio samples must be contiguous along the last dimension")
        return audio.shape[1], (audio.stride(0) if audio.shape[1] > 0 else 0), audio.dtype == torch.float32

    # ------------------------------------------------------------------ operations
    def reset(self, stream_ids=None):
        """Fresh frontend + zero rings for all streams (None) or for the given stream ids (a host sequence, or a CUDA int32
        tensor -- e.g. the streams a detection kernel just flagged; no host round trip).  A constant number of launches
        whatever the length of the list: streams join / leave a live handle without disturbing the others."""
        if stream_ids is None:
            _lib.check(self._h, self._L.mww_reset(self._h, None, 0, self._cu_stream()))
            return
        torch = _torch()
        if isinstance(stream_ids, torch.Tensor) and stream_ids.is_cuda:
            if stream_ids.dtype != torch.int32 or stream_ids.dim() != 1 or not stream_ids.is_contiguous():
                raise ValueError("device stream ids must be a contiguous 1-D CUDA int32 tensor")
            _lib.check(self._h, self._L.mww_reset_device_ids(self._h, stream_ids.data_ptr(), stream_ids.numel(), self._cu_stream()))
            return
        ids = np.ascontiguousarray(stream_ids, np.int32).reshape(-1)
        _lib.check(self._h, self._L.mww_reset(self._h, ids.ctypes.data, ids.size, self._cu_stream()))

    def set_window_step(self, hop_samples: int):
        """window_step of the frontend in samples (mww_set_window_step): 160 = the 10 ms pymicro_features hard-wires (default),
        320 = the 20 ms default of the TF-op path (audio_utils.py:29,73).  Only while no samples are buffered."""
        _lib.check(self._h, self._L.mww_set_window_step(self._h, int(hop_samples)))
        self.hop = int(hop_samples)

    def reset_frontend(self):
        _lib.check(self._h, self._L.mww_reset_frontend(self._h, self._cu_stream()))

    def features(self, audio, out=None):
        """int16 or float32 CUDA tensor [S, N] -> uint16 CUDA tensor [S, rows, 40] (rows may be 0); `out` reuses a caller buffer."""
        torch = _torch()
        n, stride, is_f32 = self._check_audio(audio)
        rows = max((self.frontend_buffered + n - WINDOW) // self.hop + 1, 0) if self.frontend_buffered + n >= WINDOW else 0
        if out is None:
            out = torch.empty((self.n_streams, max(rows, 1), NUM_FEATURES), dtype=torch.uint16, device=self._dev())
        elif (out.dtype != torch.uint16 or not out.is_cuda or not out.is_contiguous() or out.dim() != 3 or out.shape[0] != self.n_streams
              or out.shape[1] < max(rows, 1) or out.shape[2] != NUM_FEATURES):
            raise ValueError("out must be a contiguous CUDA uint16 tensor [n_streams, >= rows, 40]")
        got = ctypes.c_int(0)
        fn = self._L.mww_features_f32 if is_f32 else self._L.mww_features
        _lib.check(self._h, fn(self._h, audio.data_ptr(), n, max(stride, n), out.data_ptr(), out.shape[1], ctypes.byref(got), self._cu_stream()))
        return out[:, :got.value]

    def infer(self, rows):
        """feature rows [S, R, 40] (uint16 / float32 / int8 CUDA tensor) -> float32 probabilities [S, steps]."""
        torch = _torch()
        kinds = {torch.uint16: _lib.MWW_ROWS_U16, torch.float32: _lib.MWW_ROWS_F32, torch.int8: _lib.MWW_ROWS_I8}
        if rows.dtype not in kinds or rows.dim() != 3 or rows.shape[0] != self.n_streams or rows.shape[2] != NUM_FEATURES or not rows.is_cuda:
            raise ValueError("rows must be a CUDA uint16/float32/int8 tensor of shape [n_streams, R, 40]")
        rows = rows.contiguous()
        r = rows.shape[1]
        steps = (self.pending_rows + r) // self.stride
        probs = torch.empty((self.n_streams, max(steps, 1)), dtype=torch.float32, device=self._dev())
        got = ctypes.c_int(0)
        _lib.check(self._h, self._L.mww_infer_features(self._h, rows.data_ptr(), kinds[rows.dtype], r, max(r, 0), probs.data_ptr(),
                                                       max(steps, 1), ctypes.byref(got), self._cu_stream()))
        return probs[:, :got.value]

    def infer_strided(self, rows_ptr: int, row_type: int, n_rows: int, rows_stride: int, probs_ptr: int, max_probs: int) -> int:
        """mww_infer_features on raw device pointers: stream s reads n_rows rows at rows_ptr + s * rows_stride rows and
        writes its probabilities at probs_ptr + s * max_probs.  Returns the steps run.  For callers that lay the rows of
        all streams out in one buffer themselves (Model.predict_spectrograms)."""
        got = ctypes.c_int(0)
        _lib.check(self._h, self._L.mww_infer_features(self._h, ctypes.c_void_p(int(rows_ptr)), int(row_type), int(n_rows), int(rows_stride),
                                                       ctypes.c_void_p(int(probs_ptr)), int(max_probs), ctypes.byref(got), self._cu_stream()))
        return got.value

    def copy_nn_state(self, dst_ids, src: "StreamEngine", src_ids) -> None:
        """Stream dst_ids[i] of this engine takes the NN ring state of stream src_ids[i] of `src` (same model, same
        device, no pending rows), device to device and ordered on the current CUDA stream (mww_copy_nn_state)."""
        d = np.ascontiguousarray(dst_ids, np.int32).reshape(-1)
        s = np.ascontiguousarray(src_ids, np.int32).reshape(-1)
        if d.size != s.size:
            raise ValueError("dst_ids and src_ids must have the same length")
        _lib.check(self._h, self._L.mww_copy_nn_state(self._h, d.ctypes.data, src._h, s.ctypes.data, d.size, self._cu_stream()))

    def predict_clip(self, audio, out=None):
        """int16 or float32 CUDA tensor [S, N] -> float32 probabilities [S, steps]; state carries over between calls.  float32
        samples are converted to int16 inside the frontend kernels (x * 32768, clipped, as audio_utils.to_int16)."""
        torch = _torch()
        n, stride, is_f32 = self._check_audio(audio)
        buffered = self.frontend_buffered
        rows = (buffered + n - WINDOW) // self.hop + 1 if buffered + n >= WINDOW else 0
        steps = (self.pending_rows + rows) // self.stride
        if out is None:
            out = torch.empty((self.n_streams, max(steps, 1)), dtype=torch.float32, device=self._dev())
        got = ctypes.c_int(0)
        fn = self._L.mww_predict_clip_f32 if is_f32 else self._L.mww_predict_clip
        _lib.check(self._h, fn(self._h, audio.data_ptr(), n, max(stride, n), out.data_ptr(), out.shape[1], ctypes.byref(got), self._cu_stream()))
        return out[:, :got.value]

    step = predict_clip  # the live "one chunk of new audio per call" surface (north_star step())

    def predict_clip_host(self, audio: np.ndarray, out: np.ndarray | None = None) -> np.ndarray:
        """int16 HOST array [S, N] -> float32 HOST array [S, steps]; copies are pipelined inside the library."""
        if audio.dtype != np.int16 or audio.ndim != 2 or audio.shape[0] != self.n_streams:
            raise ValueError("audio must be an int16 array of shape [n_streams=%d, n_samples]" % self.n_streams)
        if audio.strides[1] != 2 and audio.shape[1] > 1:
            audio = np.ascontiguousarray(audio)
        n = audio.shape[1]
        buffered = self.frontend_buffered
        rows = (buffered + n - WINDOW) // self.hop + 1 if buffered + n >= WINDOW else 0
        steps = (self.pending_rows + rows) // self.stride
        if out is None:
            out = np.empty((self.n_streams, max(steps, 1)), np.float32)
        got = ctypes.c_int(0)
        _lib.check(self._h, self._L.mww_predict_clip_host(self._h, audio.ctypes.data, n, audio.strides[0] // 2 if n else 0, out.ctypes.data,
                                                          out.shape[1], ctypes.byref(got)))
        return out[:, :got.value]

    def predict_clip_remote(self, src_ptr: int, n_samples: int, stride: int | None = None, tiles: int = 0, out=None):
        """Audio int16 [S, n_samples] at address `src_ptr` -- device memory of a PEER GPU mapped into this process
        (sharding.IngestBuffer.block_ptr) or host memory (mww_predict_clip_remote).  tiles = 0: a peer-mapped (or local) buffer
        is read in place by the frontend kernel, over NVLink; host memory is staged in 16 tiles.  tiles > 0: always staged --
        this GPU's copy engine pulls tile t+1 while tile t computes.  Returns float32 CUDA probabilities [S, steps];
        stream-ordered like predict_clip."""
        torch = _torch()
        n = int(n_samples)
        buffered = self.frontend_buffered
        rows = (buffered + n - WINDOW) // self.hop + 1 if buffered + n >= WINDOW else 0
        steps = (self.pending_rows + rows) // self.stride
        if out is None:
            out = torch.empty((self.n_streams, max(steps, 1)), dtype=torch.float32, device=self._dev())
        elif out.dtype != torch.float32 or not out.is_cuda or not out.is_contiguous() or out.dim() != 2 or out.shape[0] != self.n_streams:
            raise ValueError("out must be a contiguous CUDA float32 tensor [n_streams, >= steps]")
        got = ctypes.c_int(0)
        _lib.check(self._h, self._L.mww_predict_clip_remote(self._h, ctypes.c_void_p(int(src_ptr)), n, int(stride) if stride else n, out.data_ptr(),
                                                           out.shape[1], ctypes.byref(got), int(tiles), self._cu_stream()))
        return out[:, :got.value]

    # ------------------------------------------------------------------ pinned host buffers next to the GPU
    def host_buffer(self, shape, dtype=np.int16, write_combined: bool = False) -> np.ndarray:
        """Pinned host array on the NUMA node this engine's GPU hangs off (mww_host_alloc): full-rate predict_clip_host copies
        on a two-socket box whatever CPU the caller runs on.  Freed when the array (and every view of it) is gone."""
        return host_array(shape, dtype, self.device, write_combined)

    # ------------------------------------------------------------------ per-kernel device timing
    KERNEL_CLASSES = ("k1_spectral", "k2_temporal", "mixednet", "carry_update")

    def profile(self, on: bool) -> None:
        _lib.check(self._h, self._L.mww_profile_enable(self._h, int(bool(on))))

    def profile_read(self) -> dict:
        """{class: (total_ms, launches)} accumulated since the last read (synchronises the device)."""
        ms = (ctypes.c_double * 4)(0, 0, 0, 0)
        cnt = (ctypes.c_longlong * 4)(0, 0, 0, 0)
        _lib.check(self._h, self._L.mww_profile_read(self._h, ms, cnt))
        return {k: (float(ms[i]), int(cnt[i])) for i, k in enumerate(self.KERNEL_CLASSES)}

    def timeline_read(self, max_tiles: int = 256) -> np.ndarray:
        """[tiles, 4] float32 ms (copy start, copy end, kernels start, kernels end; relative to tile 0's copy start) of the
        most recent staged call made while profile(True) -- predict_clip_host / predict_clip_remote from a peer or host source."""
        buf = (ctypes.c_float * (4 * max_tiles))()
        n = ctypes.c_int32(0)
        _lib.check(self._h, self._L.mww_timeline_read(self._h, buf, max_tiles, ctypes.byref(n)))
        return np.ctypeslib.as_array(buf).reshape(max_tiles, 4)[:min(n.value, max_tiles)].copy()

    # ------------------------------------------------------------------ state (checkpoint / tests)
    def state_dict(self) -> dict:
        S = self.n_streams
        nn_dtype = np.int8 if self.is_quantized else np.float32
        d = dict(carry=np.zeros((S, WINDOW), np.int16), estimate=np.zeros((S, NUM_FEATURES), np.uint32))
        if self._blob is not None:
            d["nn"] = np.zeros((S, self.state_elements), nn_dtype)
            d["pending"] = np.zeros((S, max(self.stride - 1, 1), NUM_FEATURES), nn_dtype)
        _lib.check(self._h, self._L.mww_get_state(self._h, d["carry"].ctypes.data, d["estimate"].ctypes.data,
                                                  d["nn"].ctypes.data if "nn" in d else None,
                                                  d["pending"].ctypes.data if "pending" in d else None))
        info = self._info()
        d["frontend_buffered"] = info.frontend_buffered
        d["pending_rows"] = info.pending_rows
        return d

    def load_state_dict(self, d: dict) -> None:
        nn_dtype = np.int8 if self.is_quantized else np.float32
        carry = np.ascontiguousarray(d["carry"], np.int16)
        est = np.ascontiguousarray(d["estimate"], np.uint32)
        nn = np.ascontiguousarray(d["nn"], nn_dtype) if "nn" in d else None
        pend = np.ascontiguousarray(d["pending"], nn_dtype) if "pending" in d else None
        _lib.check(self._h, self._L.mww_set_state(self._h, carry.ctypes.data, int(d["frontend_buffered"]), est.ctypes.data,
                                                  nn.ctypes.data if nn is not None else None, pend.ctypes.data if pend is not None else None,
                                                  int(d.get("pending_rows", 0))))
