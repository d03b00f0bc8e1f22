"""Drop-in for ``microwakeword.inference`` (reference: microwakeword/inference.py:25-170).

Same class, same methods, same argument meaning and return types; the arithmetic runs in the
sm_90a kernels of libmww_b200.so instead of tf.lite.Interpreter + pymicro_features.

Differences that are deliberate and documented (SURVEY.md Appendix D):
  * the model file is an MWW container (microwakeword_b200/model_file.py), not a .tflite flatbuffer --
    no TensorFlow / flatbuffers / .tflite exists in this environment to build or validate a reader;
  * ``predict_clip`` works (the reference raises TypeError at inference.py:78 because it passes
    ``stride_ms=`` to a function whose parameter is ``step_ms``); the frontend hop is the 10 ms that
    pymicro_features hard-wires -- ``step_ms`` is accepted and ignored exactly like the reference's
    default ``use_c=True`` path ignores it (audio_utils.py:50-64);
  * optional ``batch`` / ``device`` keyword arguments expose the many-stream engine
    (``step`` / ``reset``); with the defaults the object behaves as the reference's single-stream Model.
"""

from __future__ import annotations

import numpy as np

from .audio.audio_utils import clip_samples_fed, to_int16
from .engine import StreamEngine
from .model_file import FEATURE_SCALE, NUM_FEATURES


class Model:
    """
    Class for loading and running microwakeword streaming models on an H100

    Args:
        tflite_model_path (str | bytes): Path to (or bytes of) a streaming ``.tflite`` model (microwakeword_b200/tflite_file.py)
            or an MWW model container (microwakeword_b200/model_file.py).
        stride (int | None, optional): Time dimension's stride. If None, then the stride is the input tensor's time dimension. Defaults to None.
        batch (int): number of independent streams carried by this object (extension; default 1).
        device (int): CUDA device index (extension; default 0).
    """

    def __init__(self, tflite_model_path, stride: int | None = None, *, batch: int = 1, device: int = 0):
        self.engine = StreamEngine(tflite_model_path, n_streams=batch, device=device)
        info = self.engine.info
        self.is_quantized_model = bool(info.is_quantized)                       # inference.py:44
        self.input_feature_slices = int(info.input_feature_slices)             # inference.py:45
        self.stride = self.input_feature_slices if stride is None else stride  # inference.py:47-50
        in_dtype = np.int8 if self.is_quantized_model else np.float32
        out_dtype = np.uint8 if self.is_quantized_model else np.float32
        # the dictionaries tf.lite's get_input_details()/get_output_details() would return (inference.py:41-42)
        self.input_details = [{
            "name": "input", "index": 0, "shape": np.array([1, self.input_feature_slices, NUM_FEATURES], np.int32), "dtype": in_dtype,
            "quantization": (float(info.input_scale), int(info.input_zero_point)),
            "quantization_parameters": {"scales": np.array([info.input_scale], np.float32),
                                        "zero_points": np.array([info.input_zero_point], np.int32), "quantized_dimension": 0},
        }]
        self.output_details = [{
            "name": "output", "index": 1, "shape": np.array([1, 1], np.int32), "dtype": out_dtype,
            "quantization": (float(info.output_scale), int(info.output_zero_point)),
            "quantization_parameters": {"scales": np.array([info.output_scale], np.float32),
                                        "zero_points": np.array([info.output_zero_point], np.int32), "quantized_dimension": 0},
        }]
        self.model = self.engine  # the reference keeps the interpreter here (inference.py:64)

    # ------------------------------------------------------------------ reference surface
    def predict_clip(self, data: np.ndarray, step_ms: int = 20):
        """Run the model on a single clip of audio data

        Args:
            data (numpy.ndarray): input data for the model (16 khz, 16-bit PCM audio data)
            step_ms (int): accepted for signature compatibility; the frontend hop is 10 ms (see module docstring).

        Returns:
            list: model predictions for the input audio data
        """
        self._single()
        torch = _torch()
        audio = to_int16(np.asarray(data)).reshape(-1)
        fed = clip_samples_fed(audio.size)                       # strict '<' loop, audio_utils.py:56
        self.engine.reset_frontend()                             # fresh MicroFrontend per clip, audio_utils.py:52
        if fed == 0:
            return []
        dev = torch.from_numpy(np.ascontiguousarray(audio[:fed])).to(self.engine._dev()).unsqueeze(0)
        spectrogram = self.engine.features(dev)                  # uint16 [1, T, 40]
        return self._predict_rows(spectrogram)

    def predict_spectrogram(self, spectrogram: np.ndarray):
        """Run the model on a single spectrogram

        Args:
            spectrogram (numpy.ndarray): Input spectrogram.

        Returns:
            list: model predictions for the input audio data
        """
        self._single()
        torch = _torch()
        rows = self._chunk_rows(spectrogram)
        if rows.shape[0] == 0:
            return []
        dev = torch.from_numpy(rows.view(np.int16) if rows.dtype == np.uint16 else rows).to(self.engine._dev())
        if rows.dtype == np.uint16:
            dev = dev.view(torch.uint16)
        return self._predict_rows(dev.unsqueeze(0))

    def predict_spectrograms(self, spectrograms, max_streams: int = 65536):
        """``[self.predict_spectrogram(s) for s in spectrograms]`` -- same probabilities, same list-of-np.float32 type,
        same state afterwards -- computed in one batched pass over up to `max_streams` streams (microwakeword_b200.batched).

        This is the loop the reference's evaluation harness runs (test.py:335-367, :452-454): one interpreter, never reset,
        so every track starts from the state the previous one left.  Int8 models give bit-identical probabilities and
        state; fp32 ones agree to rounding (the batched pass may use a different kernel for a call than a per-track call).
        Pre-quantised int8 tracks cannot be mixed with tracks of other dtypes (ValueError).

        The pass keeps two things on the Model for the next call: a pinned host buffer the size of the largest test set
        uploaded so far, and an engine of as many streams as the last plan used (its NN state: up to 65 536 x 16.7 KB
        for fp32 okay_nabu).  release_batched() frees both."""
        flat, offsets, lengths = self._predict_spectrograms_device(spectrograms, max_streams)
        host = flat.cpu().numpy()
        return [list(host[o:o + n]) for o, n in zip(offsets, lengths)]

    def release_batched(self):
        """Free the pinned upload buffer and the batched engine predict_spectrograms keeps between calls; the next call
        allocates them again."""
        done = getattr(self, "_staging_done", None)
        if done is not None:
            done.synchronize()
        eng = getattr(self, "_pe_engine", None)
        if eng is not None:
            eng.close()
        self._pe_engine = self._staging_buf = self._staging_done = None

    def quantize_input_data(self, data: np.ndarray, input_details: dict) -> np.ndarray:
        """quantize the input data using scale and zero point (inference.py:127-147: truncating astype, no clamp)"""
        data_type = input_details["dtype"]
        q = input_details["quantization_parameters"]
        input_scale, input_zero_point = q["scales"][0], q["zero_points"][0]
        data = np.asarray(data, np.float32) / np.float32(input_scale) + np.float32(input_zero_point)
        return data.astype(np.int32).astype(data_type)            # C-style wrap made explicit (numpy's float->int8 is undefined out of range)

    def dequantize_output_data(self, data: np.ndarray, output_details: dict) -> np.ndarray:
        """Dequantize the model output (inference.py:149-170: hard-coded 255)"""
        output_zero_point = output_details["quantization_parameters"]["zero_points"][0]
        output_scale = 255.0
        return 1 / output_scale * (np.asarray(data).astype(np.float32) - output_zero_point)

    # ------------------------------------------------------------------ many-stream extension (north_star step surface)
    def step(self, audio):
        """Feed new audio for every stream: int16 [batch, n] (numpy or CUDA tensor; a CUDA tensor may also be float32 in [-1, 1],
        converted on the GPU as to_int16 converts it) -> probabilities [batch, steps].
        n is typically 480 (one 30 ms model step); state carries over between calls."""
        torch = _torch()
        if isinstance(audio, np.ndarray):
            return self.engine.predict_clip_host(np.ascontiguousarray(to_int16(audio)))
        return self.engine.predict_clip(audio)

    def reset(self, stream_ids=None):
        self.engine.reset(stream_ids)

    def _arch(self):
        """MixedNet hyper-parameters of the loaded model (the container's `arch` tensor)."""
        if getattr(self, "_arch_cache", None) is None:
            from . import model_file as MF
            self._arch_cache = MF.Arch.decode(MF.read_container(self.engine._blob)["arch"])
        return self._arch_cache

    def nonstreaming_length(self) -> int:
        """Rows of the shortest window the non-streaming graph accepts = its receptive field (model_train_eval.py:64-88 run
        backwards): every ring and the head window filled with real data.  203 for okay_nabu (the reference trains on 204-row windows)."""
        a = self._arch()
        span = sum(a.block_ring_rows(i) for i in range(a.n_blocks)) + a.head_rows - 1
        return a.first_conv_kernel_size + a.stride * span

    def predict_nonstreaming(self, spectrograms: np.ndarray, batch_size: int = 1024) -> np.ndarray:
        """Batched NON-streaming evaluation (SURVEY.md 8 f-4; what the reference's Keras model computes on
        `[batch, spectrogram_length, 40]` windows in train.py:41-163 with batch_size=1024): one probability per window.

        Every conv of the graph is 'valid', so the non-streaming output equals the streaming model's LAST step once every
        ring holds real data (README.md:27-28).  The streaming first conv keeps k0 - stride rows of history
        (stream.py:253-255), so step j reads rows [j s - (k0 - s), (j + 1) s): d = (-(k0 - s)) mod s leading rows are
        prepended to put the steps on the non-streaming positions (d = 1 for okay_nabu), and trailing rows the strided
        'valid' conv would not reach are dropped.  Works for every geometry the engine loads, float or int8 (for a quantised
        model this is the int8 streaming graph's last step: float rows are quantised on load, inference.py:127-147).
        Windows go through a persistent engine of `batch_size` streams (the reference's evaluate batch)."""
        import torch
        x = np.asarray(spectrograms)
        if x.ndim != 3 or x.shape[2] != NUM_FEATURES:
            raise ValueError("spectrograms must have shape [batch, T, 40]")
        a = self._arch()
        k0, s = a.first_conv_kernel_size, a.stride
        b, t = x.shape[0], x.shape[1]
        if t < self.nonstreaming_length():
            raise ValueError("window shorter than the model's receptive field (%d rows)" % self.nonstreaming_length())
        if x.dtype == np.uint16:
            x = x.astype(np.float32) * np.float32(FEATURE_SCALE)
        x = np.ascontiguousarray(x, np.float32)
        d = (-(k0 - s)) % s
        t_used = k0 + s * ((t - k0) // s)                        # rows the strided 'valid' first conv reaches
        steps = (t_used + d) // s
        cap = max(1, min(int(batch_size), b))
        eng = getattr(self, "_ns_engine", None)
        if eng is None or eng.n_streams != cap:
            if eng is not None:
                eng.close()
            eng = self._ns_engine = StreamEngine(self.engine._blob, n_streams=cap, device=self.engine.device)
        out = np.empty(b, np.float32)
        rows = np.zeros((cap, t_used + d, NUM_FEATURES), np.float32)
        for first in range(0, b, cap):
            n = min(cap, b - first)
            rows[:n, d:] = x[first:first + n, :t_used]
            eng.reset()                                           # every window starts from zero rings, like a fresh Keras call
            probs = eng.infer(torch.from_numpy(rows).to(eng._dev()))
            out[first:first + n] = probs[:n, steps - 1].cpu().numpy()
        return out

    # ------------------------------------------------------------------ helpers
    def _chunk_rows(self, spectrogram) -> np.ndarray:
        """One track -> the rows predict_spectrogram feeds, [steps * input_feature_slices, 40] (inference.py:93-105)."""
        spectrogram = np.asarray(spectrogram)
        if spectrogram.ndim != 2 or spectrogram.shape[1] != NUM_FEATURES:
            raise ValueError("spectrogram must have shape [T, %d]" % NUM_FEATURES)
        # inference.py:93-96 dtype normalisation.  uint16 rows are scaled by 0.0390625 on load in the kernel.
        if np.issubdtype(spectrogram.dtype, np.uint16):
            pass
        elif spectrogram.dtype == np.int8 and self.is_quantized_model:
            pass                                                  # already quantised: inference.py:110 skips quantisation
        elif spectrogram.dtype != np.float32:
            spectrogram = spectrogram.astype(np.float32)
        # inference.py:98-105 chunking; each chunk = one invoke
        slices = self.input_feature_slices
        n_chunks = len(range(slices, len(spectrogram) + 1, self.stride))
        if self.stride == slices:
            return np.ascontiguousarray(spectrogram[:n_chunks * slices])
        idx = (np.arange(n_chunks) * self.stride)[:, None] + np.arange(slices)[None, :]
        return np.ascontiguousarray(spectrogram[idx.reshape(-1)])

    def _predict_spectrograms_device(self, spectrograms, max_streams: int = 65536):
        """predict_spectrograms with the probabilities left on the GPU: (float32 CUDA tensor, int64 offsets, int32
        lengths); track k's probabilities are flat[offsets[k] : offsets[k] + lengths[k]].  The detection kernels read
        them there (detection.streaming_model_roc, evaluation.tflite_model_accuracy)."""
        from . import _lib, batched
        torch = _torch()
        self._single()
        if int(max_streams) < 1:
            raise ValueError("max_streams must be >= 1")
        tracks = [self._chunk_rows(s) for s in spectrograms]
        slices = self.input_feature_slices
        lengths = np.asarray([t.shape[0] // slices for t in tracks], np.int32)
        dev = self.engine._dev()
        if any(t.shape[0] for t in tracks) and self.engine.pending_rows:
            raise RuntimeError("engine holds pending rows from step(); call reset() before predict_spectrogram")
        kinds = {t.dtype for t in tracks if t.shape[0]}
        if np.dtype(np.int8) in kinds and len(kinds) > 1:
            raise ValueError("predict_spectrograms: pre-quantised int8 tracks cannot be mixed with tracks of other dtypes")
        # the narrowest exact row type: uint16 -> float32 is exact (x * 0.0390625 = x * 5 / 128 fits float32's mantissa)
        if kinds == {np.dtype(np.uint16)}:
            dtype, row_type = np.uint16, _lib.MWW_ROWS_U16
        elif kinds == {np.dtype(np.int8)}:
            dtype, row_type = np.int8, _lib.MWW_ROWS_I8
        else:
            dtype, row_type = np.float32, _lib.MWW_ROWS_F32
        a = self._arch()
        p = batched.plan(lengths, slices, slices * batched.warmup_steps(a), max_streams)
        n = p.total_steps
        if n == 0:
            return torch.zeros(1, dtype=torch.float32, device=dev)[:0], p.track_offsets, lengths   # a real pointer for the kernels
        # Int8 model kernels need 16-byte aligned row pointers: with int8 rows (40 bytes) every pointer below must sit an
        # even number of rows from the buffer start.  One extra warm-up / replay step keeps it so; more history is exact too.
        odd_rows = (lambda steps: (steps * slices) % 2) if row_type == _lib.MWW_ROWS_I8 else (lambda steps: 0)
        s, seg = (p.n_streams, p.seg_steps) if p.n_streams > 1 else (1, n)
        warm = p.warmup_steps + odd_rows(p.warmup_steps) if s > 1 else 0
        replay = p.warmup_steps + odd_rows(n - p.warmup_steps)
        prefix = warm * slices
        total_rows = prefix + s * seg * slices
        host = self._staging(total_rows * NUM_FEATURES * np.dtype(dtype).itemsize).view(dtype)[:total_rows * NUM_FEATURES]
        host = host.reshape(total_rows, NUM_FEATURES)
        host[:prefix] = 0
        at = prefix
        for t in tracks:
            if t.shape[0]:
                host[at:at + t.shape[0]] = t if t.dtype == dtype else t.astype(np.float32) * np.float32(FEATURE_SCALE)
                at += t.shape[0]
        host[at:] = 0
        rows = torch.from_numpy(host.view(np.int16) if dtype == np.uint16 else host).to(dev, non_blocking=True)
        self._staging_done = torch.cuda.Event()
        self._staging_done.record(torch.cuda.current_stream(dev))
        row_bytes = NUM_FEATURES * np.dtype(dtype).itemsize
        base = rows.data_ptr() + prefix * row_bytes
        probs = torch.empty((s, seg), dtype=torch.float32, device=dev)
        if s == 1:
            self.engine.infer_strided(base, row_type, n * slices, n * slices, probs.data_ptr(), n)
            return probs.reshape(-1), p.track_offsets, lengths
        eng = getattr(self, "_pe_engine", None)
        if eng is None or eng.n_streams != s:
            if eng is not None:
                eng.close()
            eng = self._pe_engine = StreamEngine(self.engine._blob, n_streams=s, device=self.engine.device)
        pitch = seg * slices
        scratch = torch.empty((s, max(warm, replay)), dtype=torch.float32, device=dev)
        # stream i > 0: the rows just before its segment flush whatever state it held; stream 0 takes the model's state
        eng.infer_strided(base - prefix * row_bytes, row_type, prefix, pitch, scratch.data_ptr(), warm)
        eng.copy_nn_state([0], self.engine, [0])
        eng.infer_strided(base, row_type, pitch, pitch, probs.data_ptr(), seg)
        # the model ends in the state after the last real row: that state depends only on the last `replay` steps
        self.engine.infer_strided(base + (n - replay) * slices * row_bytes, row_type, replay * slices, replay * slices,
                                  scratch.data_ptr(), replay)
        return probs.reshape(-1), p.track_offsets, lengths

    def _staging(self, nbytes: int) -> np.ndarray:
        """Pinned upload buffer of predict_spectrograms, kept between calls and grown on demand."""
        from .engine import host_array
        done = getattr(self, "_staging_done", None)
        if done is not None:
            done.synchronize()                                   # the previous upload has left the buffer
        buf = getattr(self, "_staging_buf", None)
        if buf is None or buf.size < nbytes:
            buf = self._staging_buf = host_array((max(int(nbytes), 1),), np.uint8, self.engine.device)
        return buf[:max(int(nbytes), 1)]

    def _single(self):
        if self.engine.n_streams != 1:
            raise ValueError("predict_clip / predict_spectrogram are the reference's single-stream calls; use step() with batch > 1")

    def _predict_rows(self, rows_dev):
        if rows_dev.shape[1] == 0:
            return []
        # whole chunks only, so nothing stays pending (the reference drops a trailing partial chunk, inference.py:98-105)
        if self.engine.pending_rows:
            raise RuntimeError("engine holds pending rows from step(); call reset() before predict_spectrogram")
        usable = rows_dev.shape[1] // self.input_feature_slices * self.input_feature_slices
        probs = self.engine.infer(rows_dev[:, :usable])
        return list(probs[0].cpu().numpy())                       # a Python list of np.float32, inference.py:108,123-125


def _torch():
    import torch
    return torch
