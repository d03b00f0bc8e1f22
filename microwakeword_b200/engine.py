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


def load_model_blob(model) -> bytes | None:
    """bytes of an MWW container from `model`: a path to (or bytes of) a container or a streaming ``.tflite`` flatbuffer
    (recognised and converted by ``tflite_file``, inference.py:36-45); None stays None (a frontend-only engine)."""
    if isinstance(model, (bytes, bytearray, memoryview)):
        blob = bytes(model)
    elif model is None:
        return None
    else:
        with open(model, "rb") as f:
            blob = f.read()
    from . import tflite_file
    if tflite_file.is_tflite(blob):
        blob = tflite_file.container_from_tflite(blob)      # raises TfliteError for graphs outside the hot path
    return blob


def rows_for(buffered: int, n_samples: int, hop: int) -> int:
    """feature rows a call of n_samples emits per stream when the frontend holds `buffered` samples"""
    return (buffered + n_samples - WINDOW) // hop + 1 if buffered + n_samples >= WINDOW else 0


INPUT_RATES = (8000, 16000, 22050, 24000, 32000, 44100, 48000)
RATE_PER_STREAM = _lib.MWW_RATE_PER_STREAM      # input_rate of an engine with per-stream rates (set_stream_rates)
MAX_AUDIO_HISTORY = 1 << 22                      # the largest capacity of set_audio_history, in 16 kHz samples per stream
LIVE_SAMPLES16 = 480                            # one 30 ms live call, in 16 kHz samples


G711_LAWS = {"ulaw": _lib.MWW_G711_ULAW, "alaw": _lib.MWW_G711_ALAW}     # law= of the audio calls, for uint8 G.711 audio


def _law_code(law, is_uint8: bool):
    """law= of an audio call -> the MWW_G711_* code for uint8 audio, None for int16 / float32 audio; ValueError for an
    unknown law, uint8 audio without a law, or a law with other audio"""
    if law is not None and (not isinstance(law, str) or law not in G711_LAWS):
        raise ValueError("law must be 'ulaw' or 'alaw', not %r" % (law,))
    if is_uint8 and law is None:
        raise ValueError("uint8 audio is G.711: give law='ulaw' or law='alaw'")
    if law is not None and not is_uint8:
        raise ValueError("law= is for uint8 G.711 audio, not int16 or float32")
    return None if law is None else G711_LAWS[law]


# sample formats per stream (set_stream_formats, include/mww.h): name -> code, and the bytes one sample of each code takes
SAMPLE_FORMATS = {"s16": _lib.MWW_FORMAT_S16, "ulaw": _lib.MWW_FORMAT_ULAW, "alaw": _lib.MWW_FORMAT_ALAW, "f32": _lib.MWW_FORMAT_F32}
FORMAT_BYTES = np.array([2, 1, 1, 4], np.int32)


def format_codes(formats, n: int) -> np.ndarray:
    """formats (one name of SAMPLE_FORMATS or code, or one per stream) -> np.int32 [n] codes; ValueError for anything else"""
    f = np.asarray(formats, dtype=object)
    if f.ndim == 0:
        f = np.full(n, f.item(), dtype=object)
    if f.shape != (n,):
        raise ValueError("formats must be one format per id (%d), not shape %s" % (n, f.shape))
    out = np.zeros(n, np.int32)
    for i, v in enumerate(f):
        if isinstance(v, str) and v in SAMPLE_FORMATS:
            out[i] = SAMPLE_FORMATS[v]
        elif isinstance(v, (int, np.integer)) and not isinstance(v, (bool, np.bool_)) and int(v) in SAMPLE_FORMATS.values():
            out[i] = int(v)
        else:
            raise ValueError("a sample format must be one of %s or its code 0..3, not %r" % (sorted(SAMPLE_FORMATS), v))
    return out


def bytes_for_formats(rates, formats, samples16_seen: int, n16: int) -> np.ndarray:
    """int32 [len(rates)]: the bytes row s of a mixed call of n16 holds, D_s (inputs_for_rates) times its format's sample size"""
    return inputs_for_rates(rates, samples16_seen, n16) * FORMAT_BYTES[np.asarray(formats, np.int64)]


def _kind(dtype) -> str:
    """numpy or torch sample dtype -> "int16", "float32", "uint8", ..."""
    return str(dtype).replace("torch.", "")


def _ratio(rate: int):
    from math import gcd
    g = gcd(16000, int(rate))
    return 16000 // g, int(rate) // g


def samples16(inputs_seen: int, n_samples: int, input_rate: int = 16000) -> int:
    """16 kHz samples a call of n_samples at `input_rate` yields after inputs_seen input samples (mww_set_input_rate):
    ceil((seen + n) L / M) - ceil(seen L / M) with L / M = 16000 / input_rate.  With per-stream rates (RATE_PER_STREAM)
    n_samples is n16 already."""
    if input_rate in (16000, RATE_PER_STREAM):
        return int(n_samples)
    L, M = _ratio(input_rate)
    return -(-(inputs_seen + n_samples) * L // M) + (-inputs_seen * L // M)


def rate_inputs(samples16: int, rate: int) -> int:
    """N(t, r) = floor(t M / L): the input samples a stream at `rate` has been given once the handle's counter of 16 kHz
    samples is t (mww_rate_inputs).  For even t the resampler has then emitted exactly t samples (include/mww.h)."""
    L, M = _ratio(rate)
    return int(samples16) * M // L


def inputs_for_rates(rates, samples16_seen: int, n16: int) -> np.ndarray:
    """int32 [len(rates)]: D_s = N(t + n16, r_s) - N(t, r_s), the samples row s of a call of n16 holds after t = samples16_seen"""
    rates = np.asarray(rates, np.int64)
    out = np.zeros(rates.shape, np.int32)
    for r in np.unique(rates):
        out[rates == r] = rate_inputs(samples16_seen + n16, int(r)) - rate_inputs(samples16_seen, int(r))
    return out


def resampler_history_len(rate: int) -> int:
    """input samples a stream at `rate` keeps as resampler history, H = ceil(n_taps / L) (0 at 16 kHz); for RATE_PER_STREAM
    the largest of any rate, the row length of a per-stream-rate engine's history"""
    if rate == RATE_PER_STREAM:
        return max(resampler_history_len(r) for r in INPUT_RATES)
    n, L = ctypes.c_int(0), ctypes.c_int(1)
    _lib.check(None, _lib.lib().mww_resample_taps(int(rate), None, 0, ctypes.byref(n), ctypes.byref(L), None))
    return -(-n.value // L.value)


def call_plan(buffered: int, n_samples: int, hop: int, pending_rows, strides, input_rate: int = 16000, inputs_seen: int = 0):
    """Bookkeeping of one call on a shared frontend feeding models of the given strides, each holding pending_rows[k]:
    -> (rows emitted, [steps model k runs], samples buffered after the call, [rows model k holds after the call]).
    n_samples is at `input_rate`, after `inputs_seen` input samples; the frontend sees samples16() of them.  With per-stream
    rates (input_rate RATE_PER_STREAM) n_samples is n16, which must be even, and inputs_seen is the counter t."""
    if input_rate == RATE_PER_STREAM and (int(n_samples) < 0 or int(n_samples) % 2):
        raise ValueError("with per-stream rates a call is an even number of 16 kHz samples, not %d" % n_samples)
    n16 = samples16(inputs_seen, n_samples, input_rate)
    rows = rows_for(buffered, n16, hop)
    steps = [(p + rows) // s for p, s in zip(pending_rows, strides)]
    pending = [(p + rows) % s for p, s in zip(pending_rows, strides)]
    return rows, steps, buffered + n16 - rows * hop, pending


class StreamRecords:
    """Streams exported from an engine (mww_export_streams): `data`, torch.uint8 [n, record_bytes] on the exporting
    engine's device, one packed record per stream (include/mww.h), and `layout`, the _lib.MwwStreamLayout that travels with
    them: the sizes, models and lockstep counters an importing engine must share.  `history` is None, or the last m samples
    of each stream's audio history, oldest first: a CUDA int16 tensor [n, m] that import writes back after the records.
    Records exported with resampler=True (mww_export_resampled_streams) also carry each stream's resampler history:
    `resampler` is then the _lib.MwwResamplerLayout (record size and the exporter's input-rate counters) and `rates` the
    streams' input rates, np.int32 [n]; both are None otherwise.  `formats` is None, or (records of an engine with per-stream
    rates) the streams' sample formats, np.int32 [n] codes, which import_streams gives the streams it writes."""

    _SCALARS = ("record_bytes", "n_models", "frontend_buffered", "hop_samples")
    _ARRAYS = ("pending_rows", "model_hash", "rows_are_features")
    _RESAMPLER = ("record_bytes", "resampler_off", "rate", "inputs_seen", "samples16_seen")

    def __init__(self, data, layout, history=None, resampler=None, rates=None, formats=None):
        self.data, self.layout, self.history = data, layout, history
        self.resampler, self.rates, self.formats = resampler, rates, formats

    def save(self, path) -> None:
        """np.savez of the records, the layout's fields, the history when there is one and the resampler layout and rates
        when there are: a checkpoint of some streams"""
        fields = {k: np.asarray(getattr(self.layout, k)) for k in self._SCALARS}
        fields.update({k: np.ctypeslib.as_array(getattr(self.layout, k)).copy() for k in self._ARRAYS})
        if self.history is not None:
            fields["audio_history"] = self.history.cpu().numpy()
        if self.resampler is not None:
            fields.update({"resampler_" + k: np.asarray(getattr(self.resampler, k)) for k in self._RESAMPLER})
            fields["rates"] = np.asarray(self.rates, np.int32)
        if self.formats is not None:
            fields["formats"] = np.asarray(self.formats, np.int32)
        np.savez(path, data=self.data.cpu().numpy(), **fields)

    @classmethod
    def load(cls, path, device) -> "StreamRecords":
        torch = _torch()
        layout = _lib.MwwStreamLayout()
        resampler = rates = formats = None
        with np.load(path) as z:
            for k in cls._SCALARS:
                setattr(layout, k, int(z[k]))
            for k in cls._ARRAYS:
                np.ctypeslib.as_array(getattr(layout, k))[:] = z[k]
            data = torch.from_numpy(z["data"]).to(device)
            history = torch.from_numpy(z["audio_history"]).to(device) if "audio_history" in z.files else None
            if "rates" in z.files:
                resampler = _lib.MwwResamplerLayout()
                for k in cls._RESAMPLER:
                    setattr(resampler, k, int(z["resampler_" + k]))
                rates = np.ascontiguousarray(z["rates"], np.int32)
            if "formats" in z.files:
                formats = np.ascontiguousarray(z["formats"], np.int32)
        return cls(data, layout, history, resampler, rates, formats)


class _Engine:
    """What every engine has: a handle whose `n_streams` streams share one frontend, its argument checks, resets,
    features, pinned host buffers and timing.  Subclasses create the handle and run the models."""

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
    def input_rate(self) -> int:
        return self._rate()[0]

    def _rate(self):
        """-> (input rate, input samples seen since the last reset)"""
        rate, seen = ctypes.c_int(0), ctypes.c_longlong(0)
        _lib.check(self._h, self._L.mww_get_input_rate(self._h, ctypes.byref(rate), ctypes.byref(seen)))
        return rate.value, seen.value

    def _samples16(self, n_samples: int) -> int:
        rate, seen = self._rate()
        return samples16(seen, n_samples, rate)

    def set_input_rate(self, rate: int):
        """Sample rate of the audio this engine is given (mww_set_input_rate): one of INPUT_RATES, 16000 by default.  Any other
        rate is resampled to 16 kHz on the GPU in front of the frontend; every call then takes samples at this rate.  Only
        while no samples are buffered (after create / reset / reset_frontend).  On an engine with per-stream rates it returns
        every stream to this one rate."""
        _lib.check(self._h, self._L.mww_set_input_rate(self._h, int(rate)))
        self._rate_set = self._pair_set = None

    # ------------------------------------------------------------------ per-stream input rates
    @property
    def per_stream_rates(self) -> bool:
        return self.input_rate == RATE_PER_STREAM

    @property
    def stream_rates(self) -> np.ndarray:
        """int32 [n_streams]: each stream's input rate (the engine's rate for every stream unless per_stream_rates)"""
        out = np.zeros(self.n_streams, np.int32)
        _lib.check(self._h, self._L.mww_get_stream_rates(self._h, out.ctypes.data, None))
        return out

    def set_stream_rates(self, ids, rates) -> None:
        """Stream ids[i] takes audio at rates[i] (one of INPUT_RATES; a single rate applies to every listed id), ordered on
        the current CUDA stream (mww_set_stream_rates).  The first call turns a 16 kHz engine with nothing buffered into an
        engine with per-stream rates, every stream not listed at 16 kHz.  Each listed stream's resampler history is zeroed:
        a client joining a slot calls reset(ids) as well to restart its frontend and models.  Every call then takes
        samples16= (an even number of 16 kHz samples) and row s holds inputs_for(samples16)[s] samples."""
        ids = self._ids(ids)
        r = np.asarray(rates)
        if r.ndim == 0:
            r = np.full(ids.size, int(r))
        if r.shape != ids.shape or (r.size and not np.issubdtype(r.dtype, np.integer)):
            raise ValueError("rates must be one integer rate per id")
        r = np.ascontiguousarray(r, np.int32)
        self._rate_set = self._pair_set = None
        _lib.check(self._h, self._L.mww_set_stream_rates(self._h, ids.ctypes.data, r.ctypes.data, ids.size, self._cu_stream()))

    def _rates_present(self) -> tuple:
        """the distinct stream rates, kept until the rates change (a call's row width needs them, not every stream's)"""
        if getattr(self, "_rate_set", None) is None:
            self._rate_set = tuple(int(r) for r in np.unique(self.stream_rates))
        return self._rate_set

    # ------------------------------------------------------------------ per-stream sample formats
    @property
    def stream_formats(self) -> np.ndarray:
        """int32 [n_streams]: each stream's sample format code (SAMPLE_FORMATS; "s16" for every stream unless
        per_stream_rates)"""
        out = np.zeros(self.n_streams, np.int32)
        _lib.check(self._h, self._L.mww_get_stream_formats(self._h, out.ctypes.data))
        return out

    def set_stream_formats(self, ids, formats) -> None:
        """Stream ids[i] sends its audio in formats[i] from the next call on ("s16", "f32", "ulaw", "alaw" or their codes; one
        format applies to every listed id), ordered on the current CUDA stream (mww_set_stream_formats).  Only on an engine
        with per-stream rates (MwwError MWW_EUNSUPPORTED otherwise).  No state changes: a stream may switch formats between
        any two calls.  The mixed=True calls then take uint8 rows, row s holding bytes_for(samples16)[s] bytes."""
        ids = self._ids(ids)
        f = format_codes(formats, ids.size)
        self._pair_set = None
        _lib.check(self._h, self._L.mww_set_stream_formats(self._h, ids.ctypes.data, f.ctypes.data, ids.size, self._cu_stream()))

    def _pairs_present(self) -> tuple:
        """the distinct (rate, format) pairs of the streams, kept until rates or formats change"""
        if getattr(self, "_pair_set", None) is None:
            pairs = np.unique(np.stack([self.stream_rates, self.stream_formats], 1), axis=0)
            self._pair_set = tuple((int(r), int(f)) for r, f in pairs)
        return self._pair_set

    def bytes_for(self, samples16: int) -> np.ndarray:
        """int32 [n_streams]: the bytes each stream's row holds in the next mixed=True call of samples16 (per_stream_rates
        only): inputs_for(samples16) times the sample size of the stream's format (2, 4 or 1 for s16, f32 and G.711).  The
        rows' pitch is at least the largest of these and, like the buffer's address, a multiple of 4."""
        return self.inputs_for(samples16) * FORMAT_BYTES[self.stream_formats]

    def _mixed_len(self, width: int, stride: int, ptr: int, samples16) -> int:
        """-> n_samples (n16) of a mixed=True call whose rows hold `width` bytes at pitch `stride` from address `ptr`, or
        ValueError before the library is called"""
        rate, t = self._rate()
        if rate != RATE_PER_STREAM:
            raise ValueError("mixed=True is for an engine with per-stream rates (set_stream_rates)")
        n16 = self._check_samples16(samples16)
        need = max((int(bytes_for_formats([r], [f], t, n16)[0]) for r, f in self._pairs_present()), default=0) if n16 else 0
        if width < need:
            raise ValueError("mixed rows hold %d bytes; this call of %d 16 kHz samples needs %d (bytes_for)" % (width, n16, need))
        if stride % 4 or ptr % 4:
            raise ValueError("mixed rows need an address and a row pitch that are multiples of 4 bytes (pitch %d)" % stride)
        return n16

    def inputs_for(self, samples16: int) -> np.ndarray:
        """int32 [n_streams]: the samples each stream's row holds in the next call of samples16 (per_stream_rates only):
        D_s = N(t + samples16, r_s) - N(t, r_s), N(t, r) = floor(t M / L)"""
        rate, t = self._rate()
        if rate != RATE_PER_STREAM:
            raise ValueError("inputs_for is for an engine with per-stream rates (set_stream_rates)")
        n16 = self._check_samples16(samples16)
        return inputs_for_rates(self.stream_rates, t, n16)

    @staticmethod
    def _check_samples16(samples16) -> int:
        if samples16 is None or int(samples16) != samples16 or int(samples16) < 0 or int(samples16) % 2:
            raise ValueError("with per-stream rates every call needs samples16=, an even number of 16 kHz samples >= 0 (got %r)"
                             % (samples16,))
        return int(samples16)

    def _call_len(self, width: int, samples16) -> int:
        """-> n_samples for the library.  One input rate: the audio's width (samples16 must be None).  Per-stream rates: the
        checked samples16, once the rows (`width` samples) are known to hold every stream's D_s."""
        rate, t = self._rate()
        if rate != RATE_PER_STREAM:
            if samples16 is not None:
                raise ValueError("samples16= is for an engine with per-stream rates (set_stream_rates)")
            return int(width)
        n16 = self._check_samples16(samples16)
        need = int(inputs_for_rates(self._rates_present(), t, n16).max()) if n16 and self.n_streams else 0
        if width < need:
            raise ValueError("audio rows hold %d samples; this call of %d 16 kHz samples needs %d (inputs_for)" % (width, n16, need))
        return n16

    def resampler_history(self) -> int:
        """input samples each stream keeps as resampler history (0 at 16 kHz; with per-stream rates the row length H_max)"""
        return resampler_history_len(self.input_rate)

    def _get_resampler(self, d: dict) -> None:
        """the resampler's part of state_dict (nothing at 16 kHz)"""
        if self.input_rate == 16000:
            return
        hist = np.zeros((self.n_streams, self.resampler_history()), np.int16)
        seen = ctypes.c_longlong(0)
        _lib.check(self._h, self._L.mww_get_resampler_state(self._h, hist.ctypes.data, ctypes.byref(seen)))
        d.update(input_rate=self.input_rate, resampler_history=hist, inputs_seen=seen.value)
        if self.input_rate == RATE_PER_STREAM:
            d["stream_rates"] = self.stream_rates
            d["stream_formats"] = self.stream_formats

    def _set_resampler(self, d: dict) -> None:
        rate = int(d.get("input_rate", 16000))
        if rate != self.input_rate and not (rate == RATE_PER_STREAM and self.input_rate == 16000):
            raise ValueError("the state was taken at %d Hz, this engine runs at %d Hz" % (rate, self.input_rate))
        if rate == 16000:
            return
        hist = np.ascontiguousarray(d["resampler_history"], np.int16)
        if hist.shape != (self.n_streams, resampler_history_len(rate)):
            raise ValueError("resampler_history must be int16 [n_streams, %d]" % resampler_history_len(rate))
        if rate == RATE_PER_STREAM:
            # the rates first (an engine at 16 kHz enters the mode), then the histories and the counter
            rates = np.ascontiguousarray(d["stream_rates"], np.int32)
            if rates.shape != (self.n_streams,):
                raise ValueError("stream_rates must be int32 [n_streams]")
            self.set_stream_rates(np.arange(self.n_streams, dtype=np.int32), rates)
            if "stream_formats" in d:
                self.set_stream_formats(np.arange(self.n_streams, dtype=np.int32), np.ascontiguousarray(d["stream_formats"], np.int32))
        _lib.check(self._h, self._L.mww_set_resampler_state(self._h, hist.ctypes.data, int(d["inputs_seen"])))

    @property
    def launch_count(self) -> int:
        return int(self._L.mww_launch_count(self._h))

    @staticmethod
    def _check_mixed(law, mixed: bool, is_uint8: bool) -> bool:
        """mixed=True: the audio is uint8 rows of bytes in each stream's format, and law= has no meaning"""
        if not mixed:
            return False
        if law is not None:
            raise ValueError("law= is for uint8 audio of one G.711 law; with mixed=True each stream's format says how to read it")
        if not is_uint8:
            raise ValueError("mixed=True takes uint8 rows of bytes (bytes_for), not another dtype")
        return True

    def _check_audio(self, audio, law=None, mixed=False):
        """-> (n_samples, row pitch in samples, is_float32).  float32 audio is converted to int16 inside the frontend kernels,
        exactly as audio_utils.to_int16 converts it on the host; other float dtypes are refused (float64 keeps its exact host
        conversion: rounding it to float32 first could move a sample across an integer boundary after the x 32768).  uint8
        audio is G.711 of the given law (_law_code), decoded inside the kernels."""
        torch = _torch()
        if (audio.dtype not in (torch.int16, torch.float32, torch.uint8) or audio.dim() != 2 or audio.shape[0] != self.n_streams
                or not audio.is_cuda):
            raise ValueError("audio must be a CUDA int16 or float32 tensor (uint8 with law=) of shape [n_streams=%d, n_samples]"
                             % self.n_streams)
        if not self._check_mixed(law, mixed, audio.dtype == torch.uint8):
            _law_code(law, audio.dtype == torch.uint8)
        if audio.stride(1) != 1 and audio.shape[1] > 1:
            raise ValueError("audio samples must be contiguous along the last dimension")
        return audio.shape[1], (audio.stride(0) if audio.shape[1] > 0 else 0), audio.dtype == torch.float32

    def _check_host_audio(self, audio: np.ndarray, law=None, mixed=False):
        """int16 or float32 host audio [S, N] -> (the array with contiguous samples, its row pitch in samples, is_float32).
        An array whose samples are not contiguous, or whose row stride is not a whole number of samples >= N (a view made
        with as_strided or an explicit strides= argument, a broadcast, reversed rows), is copied first.  float32 goes through
        the staged pipeline as it is and is converted on the GPU as _check_audio describes; float64, other dtypes and wrong
        shapes raise ValueError here, before the library is called, as they do on the device path.  uint8 is G.711 audio of
        the given law, as on the device path."""
        if (not isinstance(audio, np.ndarray) or audio.dtype not in (np.int16, np.float32, np.uint8) or audio.ndim != 2
                or audio.shape[0] != self.n_streams):
            raise ValueError("audio must be an int16 or float32 array (uint8 with law=) of shape [n_streams=%d, n_samples]"
                             % self.n_streams)
        if not self._check_mixed(law, mixed, audio.dtype == np.uint8):
            _law_code(law, audio.dtype == np.uint8)
        n, size = audio.shape[1], audio.itemsize
        if n > 0 and ((audio.strides[1] != size and n > 1) or audio.strides[0] % size or audio.strides[0] < n * size):
            audio = np.ascontiguousarray(audio)
        return audio, (audio.strides[0] // audio.itemsize if n else 0), audio.dtype == np.float32

    def _remote_fn(self, dtype, name: str, law=None, mixed=False):
        """the int16, float32 or G.711 (uint8 with `law`) form of the raw-pointer entry point `name`, from a numpy (or torch)
        sample dtype; None is int16, or uint8 with mixed=True (the _mixed form)"""
        if dtype is None:
            dtype = np.uint8 if mixed else np.int16
        if str(dtype) in ("torch.int16", "torch.float32", "torch.uint8"):
            dtype = _kind(dtype)
        try:
            dt = np.dtype(dtype)
        except TypeError:
            dt = None
        if dt not in (np.dtype(np.int16), np.dtype(np.float32), np.dtype(np.uint8)):
            raise ValueError("dtype must be int16 or float32 (uint8 with law=), not %r" % (dtype,))
        return self._audio_fn(name, dt.name, law, mixed)

    def _audio_fn(self, name: str, kind: str, law=None, mixed=False):
        """the entry point `name` for audio of `kind` ("int16", "float32" or "uint8"): `name`, its _f32 form, its _g711 form
        with the law's code passed after the audio pointer, or with mixed=True its _mixed form"""
        if self._check_mixed(law, mixed, kind == "uint8"):
            return getattr(self._L, name + "_mixed")
        code = _law_code(law, kind == "uint8")
        if code is None:
            return getattr(self._L, name + "_f32" if kind == "float32" else name)
        fn = getattr(self._L, name + "_g711")
        return lambda h, audio, *rest: fn(h, audio, code, *rest)

    def _check_probs_out(self, out) -> None:
        torch = _torch()
        if out.dtype != torch.float32 or not out.is_cuda or not out.is_contiguous() or out.dim() != 2 or out.shape[0] != self.n_streams:
            raise ValueError("out must be a contiguous CUDA float32 tensor [n_streams, >= steps]")

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

    # ------------------------------------------------------------------ audio history
    def set_audio_history(self, capacity: int) -> None:
        """Keep the last `capacity` 16 kHz int16 samples of every stream on the GPU (mww_set_audio_history; the rule is in
        include/mww.h): 0 (off, the default) or a multiple of 8 in [8, 2**22].  Every stream's history starts as zeros and
        audio_samples_seen restarts at 0; a reset of a stream zeroes its history."""
        if isinstance(capacity, bool) or int(capacity) != capacity or not (capacity == 0 or (8 <= capacity <= MAX_AUDIO_HISTORY
                                                                                          and capacity % 8 == 0)):
            raise ValueError("capacity must be 0 or a multiple of 8 in [8, %d] (got %r)" % (MAX_AUDIO_HISTORY, capacity))
        _lib.check(self._h, self._L.mww_set_audio_history(self._h, int(capacity), self._cu_stream()))

    def _audio_history(self):
        cap, seen = ctypes.c_int(0), ctypes.c_longlong(0)
        _lib.check(self._h, self._L.mww_get_audio_history(self._h, ctypes.byref(cap), ctypes.byref(seen)))
        return cap.value, seen.value

    @property
    def audio_history_capacity(self) -> int:
        return self._audio_history()[0]

    @property
    def audio_samples_seen(self) -> int:
        """16 kHz samples every stream has appended since set_audio_history (resets do not clear it)"""
        return self._audio_history()[1]

    def audio_history(self, stream_ids, n_samples: int, out=None, end=None):
        """The last n_samples (<= audio_history_capacity) 16 kHz samples of each listed stream, oldest first, zero-padded on
        the left: a CUDA int16 tensor [len(ids), n_samples], ordered on the current CUDA stream (mww_read_audio_history).
        `stream_ids`: a host sequence (ids in [0, n_streams)) or a contiguous 1-D CUDA int32 tensor such as a detector's
        fired_ids, read with no host round trip (ids outside [0, n_streams), the -1 slots, give zero rows).  Read before
        reset(ids): a reset zeroes the history.  `out`: a CUDA int16 tensor [len(ids), >= n_samples] with contiguous rows.
        `end`: row i holds the samples [end[i] - n_samples, end[i]) of the history axis instead, zeros where they are not in
        the ring [audio_samples_seen - capacity, audio_samples_seen) (mww_read_audio_history_at); a host sequence or a
        contiguous 1-D CUDA int64 tensor aligned with the ids, such as a timed detector's event_samples."""
        torch = _torch()
        cap = self.audio_history_capacity
        if cap == 0:
            raise ValueError("the engine keeps no audio history (set_audio_history)")
        if isinstance(n_samples, bool) or int(n_samples) != n_samples or not 0 <= n_samples <= cap:
            raise ValueError("n_samples must be an integer in [0, %d] (got %r)" % (cap, n_samples))
        n_samples = int(n_samples)
        device_ids = isinstance(stream_ids, torch.Tensor) and stream_ids.is_cuda
        if device_ids:
            if stream_ids.dtype != torch.int32 or stream_ids.dim() != 1 or not stream_ids.is_contiguous() or stream_ids.device != self._dev():
                raise ValueError("device stream ids must be a contiguous 1-D CUDA int32 tensor on %s" % self._dev())
            n = stream_ids.numel()
        else:
            ids = self._ids(stream_ids)
            if ids.size and (ids.min() < 0 or ids.max() >= self.n_streams):
                raise ValueError("stream ids must be in [0, %d)" % self.n_streams)
            n = ids.size
        if out is None:
            out = torch.empty((n, n_samples), dtype=torch.int16, device=self._dev())
        elif (not isinstance(out, torch.Tensor) or out.dtype != torch.int16 or out.device != self._dev() or out.dim() != 2 or out.shape[0] != n
              or out.shape[1] < n_samples or (out.stride(1) != 1 and out.shape[1] > 1) or (n > 1 and out.stride(0) < n_samples)):
            raise ValueError("out must be a CUDA int16 tensor [len(ids)=%d, >= %d] with contiguous rows on %s" % (n, n_samples, self._dev()))
        stride = out.stride(0) if n > 1 else max(out.shape[1], n_samples)
        if end is not None:
            ends = self._history_ends(end, n)
            dids = stream_ids if device_ids else torch.from_numpy(ids).to(self._dev())
            _lib.check(self._h, self._L.mww_read_audio_history_at(self._h, dids.data_ptr(), ends.data_ptr(), n, n_samples, out.data_ptr(), stride,
                                                                  self._cu_stream()))
            return out[:, :n_samples]
        if device_ids:
            rc = self._L.mww_read_audio_history_device_ids(self._h, stream_ids.data_ptr(), n, n_samples, out.data_ptr(), stride, self._cu_stream())
        else:
            rc = self._L.mww_read_audio_history(self._h, ids.ctypes.data, n, n_samples, out.data_ptr(), stride, self._cu_stream())
        _lib.check(self._h, rc)
        return out[:, :n_samples]

    def _history_ends(self, end, n: int):
        """the ends of a read at positions as a CUDA int64 tensor [n] on this engine's device, or ValueError"""
        torch = _torch()
        if isinstance(end, torch.Tensor) and end.is_cuda:
            if end.dtype != torch.int64 or end.dim() != 1 or not end.is_contiguous() or end.device != self._dev() or end.numel() != n:
                raise ValueError("device ends must be a contiguous 1-D CUDA int64 tensor [len(ids)=%d] on %s" % (n, self._dev()))
            return end
        if hasattr(end, "is_cuda"):
            end = end.numpy()
        e = np.asarray(end)
        if e.shape != (n,) or (e.size and (e.dtype == bool or not np.issubdtype(e.dtype, np.integer))):
            raise ValueError("end must be one integer position per id (%d)" % n)
        return torch.from_numpy(np.ascontiguousarray(e, np.int64)).to(self._dev())

    def features(self, audio, out=None, samples16=None, law=None, mixed=False):
        """int16 or float32 CUDA tensor [S, N] -> uint16 CUDA tensor [S, rows, 40] (rows may be 0); `out` reuses a caller buffer.
        With per-stream rates: samples16= (even), and N >= every stream's inputs_for(samples16).  G.711 audio: a uint8 tensor
        of codes and law='ulaw' or 'alaw', decoded inside the kernels (include/mww.h gives the rule).  mixed=True (per-stream
        rates): a uint8 tensor of bytes, row s in stream s's format (set_stream_formats), N >= every bytes_for(samples16)."""
        torch = _torch()
        width, stride, _ = self._check_audio(audio, law, mixed)
        n = self._mixed_len(width, max(stride, width), audio.data_ptr(), samples16) if mixed else self._call_len(width, samples16)
        stride = max(stride, width)
        rows = rows_for(self.frontend_buffered, self._samples16(n), self.hop)
        if out is None:
            out = torch.empty((self.n_streams, max(rows, 1), NUM_FEATURES), dtype=torch.uint16, device=self._dev())
        elif (out.dtype != torch.uint16 or not out.is_cuda or not out.is_contiguous() or out.dim() != 3 or out.shape[0] != self.n_streams
              or out.shape[1] < max(rows, 1) or out.shape[2] != NUM_FEATURES):
            raise ValueError("out must be a contiguous CUDA uint16 tensor [n_streams, >= rows, 40]")
        got = ctypes.c_int(0)
        fn = self._audio_fn("mww_features", _kind(audio.dtype), law, mixed)
        _lib.check(self._h, fn(self._h, audio.data_ptr(), n, stride, out.data_ptr(), out.shape[1], ctypes.byref(got), self._cu_stream()))
        return out[:, :got.value]

    # ------------------------------------------------------------------ moving streams between engines
    @staticmethod
    def _ids(ids) -> np.ndarray:
        """a list, NumPy array or CPU tensor of global stream ids -> contiguous int32 array"""
        if hasattr(ids, "is_cuda"):
            if ids.is_cuda:
                raise ValueError("stream ids must be in host memory")
            ids = ids.numpy()
        a = np.asarray(ids)
        if a.ndim != 1 or (a.size and not np.issubdtype(a.dtype, np.integer)):
            raise ValueError("stream ids must be a 1-D sequence of integers")
        return np.ascontiguousarray(a, np.int32)

    def stream_layout(self) -> "_lib.MwwStreamLayout":
        """record size, models and current lockstep counters of this engine (mww_stream_layout_get; no device work)"""
        layout = _lib.MwwStreamLayout()
        _lib.check(self._h, self._L.mww_stream_layout_get(self._h, ctypes.byref(layout)))
        return layout

    def resampler_layout(self) -> "_lib.MwwResamplerLayout":
        """record size of resampled records and the current input-rate counters (mww_get_resampler_layout; no device work)"""
        layout = _lib.MwwResamplerLayout()
        _lib.check(self._h, self._L.mww_get_resampler_layout(self._h, ctypes.byref(layout)))
        return layout

    def export_streams(self, ids, history: int = 0, resampler: bool = False) -> StreamRecords:
        """The whole state (frontend and every model) of streams `ids` as packed records on this engine's device, ordered on
        the current CUDA stream in a constant number of launches (mww_export_streams).  The engine is not changed.
        `history` > 0 (at most audio_history_capacity) also reads the last `history` samples of each stream's audio history
        into records.history, on the same CUDA stream, so that the streams keep it when they move.  At 12 s a stream's
        history is 384 kB: move many streams in batches of ids, or carry only the samples still needed (what a verifier
        hears, an endpointer's lookback and the commands in progress).
        resampler=True exports records that also carry each stream's resampler history (mww_export_resampled_streams), on an
        engine at any input rate or with per-stream rates; records.resampler and records.rates say what the importer must
        match, and on an engine with per-stream rates records.formats holds the streams' sample formats.  Without it an engine
        that resamples refuses (MwwError, MWW_EUNSUPPORTED)."""
        torch = _torch()
        ids = self._ids(ids)
        if isinstance(history, bool) or not isinstance(history, (int, np.integer)) or history < 0:
            raise ValueError("history must be a non-negative integer (got %r)" % (history,))
        if history and not history <= self.audio_history_capacity:
            raise ValueError("history must be at most the audio history capacity %d (got %d)" % (self.audio_history_capacity, history))
        layout = _lib.MwwStreamLayout()
        if resampler:
            rs = _lib.MwwResamplerLayout()
            rates = np.zeros(ids.size, np.int32)
            data = torch.empty((ids.size, int(self.resampler_layout().record_bytes)), dtype=torch.uint8, device=self._dev())
            _lib.check(self._h, self._L.mww_export_resampled_streams(self._h, ids.ctypes.data, ids.size, data.data_ptr(), ctypes.byref(layout),
                                                                     ctypes.byref(rs), rates.ctypes.data, self._cu_stream()))
            formats = self.stream_formats[ids] if self.per_stream_rates else None
        else:
            rs = rates = formats = None
            data = torch.empty((ids.size, int(self.stream_layout().record_bytes)), dtype=torch.uint8, device=self._dev())
            _lib.check(self._h, self._L.mww_export_streams(self._h, ids.ctypes.data, ids.size, data.data_ptr(), ctypes.byref(layout),
                                                           self._cu_stream()))
        return StreamRecords(data, layout, self.audio_history(ids, int(history)) if history else None, rs, rates, formats)

    def import_streams(self, ids, records: StreamRecords) -> None:
        """Stream ids[i] of this engine takes the state of records.data[i] (mww_import_streams): it continues bit for bit as
        the exported stream would have.  Every other stream is untouched.  The records must be a contiguous uint8 tensor
        [len(ids), record_bytes] on this engine's device (ValueError otherwise); records that do not fit this engine's
        models or lockstep counters, duplicate or out-of-range ids: MwwError, nothing changed.  When records.history is
        not None (a CUDA int16 tensor [len(ids), m] on this engine's device, and this engine keeps a history), each
        stream's history becomes zeros followed by its row, written after the import (mww_write_audio_history).
        Records with a resampler layout (export_streams(..., resampler=True)) take mww_import_resampled_streams: stream
        ids[i] must already be at records.rates[i] here, and at the same phase of its resampler (include/mww.h), else
        MwwError naming the stream.  On an engine with per-stream rates, set them first:

            recs = src.export_streams(src_ids, history=m, resampler=True)
            dst.set_stream_rates(dst_ids, recs.rates)
            dst.import_streams(dst_ids, recs)

        Records that carry formats (records.formats) give them to the streams with set_stream_formats once the import is
        done, so that a stream that sent mu-law keeps being read as mu-law; formats other than "s16" need an engine with
        per-stream rates (ValueError before anything is imported otherwise)."""
        torch = _torch()
        ids = self._ids(ids)
        rs = getattr(records, "resampler", None)
        record_bytes = records.layout.record_bytes if rs is None else rs.record_bytes
        if rs is not None:
            rates = records.rates
            if not isinstance(rates, np.ndarray) or rates.dtype != np.int32 or rates.shape != (ids.size,):
                raise ValueError("records.rates must be an np.int32 array [len(ids)=%d]" % ids.size)
            rates = np.ascontiguousarray(rates)
        formats = getattr(records, "formats", None)
        if formats is not None:
            formats = format_codes(formats, ids.size)
            if formats.any() and not self.per_stream_rates:
                raise ValueError("records.formats holds formats other than 's16'; they need an engine with per-stream rates")
        data = records.data
        if (not isinstance(data, torch.Tensor) or data.dtype != torch.uint8 or data.dim() != 2 or data.shape[0] != ids.size
                or data.shape[1] != record_bytes or not data.is_contiguous() or data.device != self._dev()):
            raise ValueError("records.data must be a contiguous uint8 tensor [len(ids)=%d, record_bytes=%d] on %s"
                             % (ids.size, record_bytes, self._dev()))
        hist = getattr(records, "history", None)
        if hist is not None:
            if (not isinstance(hist, torch.Tensor) or hist.dtype != torch.int16 or hist.dim() != 2 or hist.shape[0] != ids.size
                    or hist.shape[1] > MAX_AUDIO_HISTORY or hist.device != self._dev()):
                raise ValueError("records.history must be an int16 tensor [len(ids)=%d, <= %d] on %s" % (ids.size, MAX_AUDIO_HISTORY, self._dev()))
            if self.audio_history_capacity == 0:
                raise ValueError("records carry audio history but the engine keeps none (set_audio_history)")
            if hist.shape[1] > 1 and hist.stride(1) != 1 or ids.size > 1 and hist.stride(0) < hist.shape[1]:
                hist = hist.contiguous()
        if rs is None:
            _lib.check(self._h, self._L.mww_import_streams(self._h, ids.ctypes.data, ids.size, data.data_ptr(), ctypes.byref(records.layout),
                                                           self._cu_stream()))
        else:
            _lib.check(self._h, self._L.mww_import_resampled_streams(self._h, ids.ctypes.data, ids.size, data.data_ptr(),
                                                                     ctypes.byref(records.layout), ctypes.byref(rs), rates.ctypes.data,
                                                                     self._cu_stream()))
        if hist is not None:
            stride = hist.stride(0) if ids.size > 1 else hist.shape[1]
            _lib.check(self._h, self._L.mww_write_audio_history(self._h, ids.ctypes.data, ids.size, hist.shape[1],
                                                                hist.data_ptr() if hist.numel() else None, stride, self._cu_stream()))
        if formats is not None and self.per_stream_rates:
            self.set_stream_formats(ids, formats)

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


class StreamEngine(_Engine):
    """`model`: path to (or bytes of) an MWW container or a streaming ``.tflite`` flatbuffer (recognised and converted by
    ``tflite_file``, inference.py:36-45), or None for a frontend-only engine."""

    def __init__(self, model, n_streams: int = 1, device: int = 0, input_rate: int = 16000, stream_rates=None,
                 stream_formats=None):
        if stream_rates is not None and input_rate != 16000:
            raise ValueError("give input_rate= or stream_rates=, not both")
        if stream_formats is not None and stream_rates is None:
            raise ValueError("stream_formats= needs stream_rates= (sample formats per stream need per-stream rates)")
        blob = load_model_blob(model)
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
        if input_rate != 16000:
            self.set_input_rate(input_rate)
        if stream_rates is not None:
            self.set_stream_rates(np.arange(self.n_streams, dtype=np.int32), stream_rates)
        if stream_formats is not None:
            self.set_stream_formats(np.arange(self.n_streams, dtype=np.int32), stream_formats)

    @property
    def pending_rows(self) -> int:
        return self._info().pending_rows

    def _steps(self, n_samples: int) -> int:
        return (self.pending_rows + rows_for(self.frontend_buffered, self._samples16(n_samples), self.hop)) // self.stride

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

    def predict_clip(self, audio, out=None, samples16=None, law=None, mixed=False):
        """int16 or float32 CUDA tensor [S, N] -> float32 probabilities [S, steps]; state carries over between calls.  float32
        samples are converted to int16 inside the frontend kernels (x * 32768, clipped, as audio_utils.to_int16).  With
        per-stream rates: samples16= (even), and N >= every stream's inputs_for(samples16).  G.711: uint8 codes with
        law='ulaw' or 'alaw' (as features).  mixed=True: uint8 rows in each stream's own format (as features)."""
        torch = _torch()
        width, stride, _ = self._check_audio(audio, law, mixed)
        n = self._mixed_len(width, max(stride, width), audio.data_ptr(), samples16) if mixed else self._call_len(width, samples16)
        stride = max(stride, width)
        steps = self._steps(n)
        if out is None:
            out = torch.empty((self.n_streams, max(steps, 1)), dtype=torch.float32, device=self._dev())
        got = ctypes.c_int(0)
        fn = self._audio_fn("mww_predict_clip", _kind(audio.dtype), law, mixed)
        _lib.check(self._h, fn(self._h, audio.data_ptr(), n, stride, out.data_ptr(), out.shape[1], ctypes.byref(got), self._cu_stream()))
        return out[:, :got.value]

    def step(self, audio, out=None, law=None, mixed=False):
        """the live "one chunk of new audio per call" surface (north_star step()): predict_clip; with per-stream rates a
        30 ms call (samples16 = 480)"""
        return self.predict_clip(audio, out, LIVE_SAMPLES16 if self.per_stream_rates else None, law=law, mixed=mixed)

    def predict_clip_host(self, audio: np.ndarray, out: np.ndarray | None = None, samples16=None, law=None, mixed=False) -> np.ndarray:
        """int16 or float32 HOST array [S, N] -> float32 HOST array [S, steps]; copies are pipelined inside the library.
        float32 samples cross PCIe as they are and are converted in the frontend kernels (as predict_clip converts them), and
        so do uint8 G.711 codes with law='ulaw' or 'alaw' (one byte per sample), and with mixed=True uint8 rows in each
        stream's own format.  Other dtypes (float64 included) and wrong shapes: ValueError; a too-small `out`: MwwError."""
        audio, stride, _ = self._check_host_audio(audio, law, mixed)
        n = self._mixed_len(audio.shape[1], stride, audio.ctypes.data, samples16) if mixed else self._call_len(audio.shape[1], samples16)
        steps = self._steps(n)
        if out is None:
            out = np.empty((self.n_streams, max(steps, 1)), np.float32)
        got = ctypes.c_int(0)
        fn = self._audio_fn("mww_predict_clip_host", _kind(audio.dtype), law, mixed)
        _lib.check(self._h, fn(self._h, audio.ctypes.data, n, stride, out.ctypes.data, out.shape[1], ctypes.byref(got)))
        return out[:, :got.value]

    def predict_clip_remote(self, src_ptr: int, n_samples: int, stride: int | None = None, tiles: int = 0, out=None, dtype=None,
                            samples16=None, law=None, mixed=False):
        """Audio [S, n_samples] of `dtype` (int16 by default, float32, or uint8 G.711 codes with law='ulaw' or 'alaw'; stride
        in samples; with mixed=True uint8 rows of n_samples bytes in each stream's own format, stride in bytes)
        at address `src_ptr` -- device memory of a PEER
        GPU mapped into this process (sharding.IngestBuffer.block_ptr) or host memory (mww_predict_clip_remote[_f32]).
        tiles = 0: a peer-mapped (or local) buffer is read in place by the frontend kernel, over NVLink; host memory is staged
        in 16 tiles.  tiles > 0: always staged -- this GPU's copy engine pulls tile t+1 while tile t computes.  Returns float32
        CUDA probabilities [S, steps]; stream-ordered like predict_clip.  With per-stream rates n_samples is the samples each
        row holds (>= every inputs_for(samples16)) and samples16= the call."""
        torch = _torch()
        fn = self._remote_fn(dtype, "mww_predict_clip_remote", law, mixed)
        width = int(n_samples)
        stride = int(stride) if stride else width
        n = self._mixed_len(width, stride, int(src_ptr), samples16) if mixed else self._call_len(width, samples16)
        steps = self._steps(n)
        if out is None:
            out = torch.empty((self.n_streams, max(steps, 1)), dtype=torch.float32, device=self._dev())
        else:
            self._check_probs_out(out)
        got = ctypes.c_int(0)
        _lib.check(self._h, fn(self._h, ctypes.c_void_p(int(src_ptr)), n, stride, out.data_ptr(), out.shape[1], ctypes.byref(got),
                               int(tiles), self._cu_stream()))
        return out[:, :got.value]

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
        self._get_resampler(d)
        return d

    def load_state_dict(self, d: dict) -> None:
        self._set_resampler(d)
        nn_dtype = np.int8 if self.is_quantized else np.float32
        carry = np.ascontiguousarray(d["carry"], np.int16)
        est = np.ascontiguousarray(d["estimate"], np.uint32)
        nn = np.ascontiguousarray(d["nn"], nn_dtype) if "nn" in d else None
        pend = np.ascontiguousarray(d["pending"], nn_dtype) if "pending" in d else None
        _lib.check(self._h, self._L.mww_set_state(self._h, carry.ctypes.data, int(d["frontend_buffered"]), est.ctypes.data,
                                                  nn.ctypes.data if nn is not None else None, pend.ctypes.data if pend is not None else None,
                                                  int(d.get("pending_rows", 0))))


class MultiModelEngine(_Engine):
    """K wake-word / VAD models over ONE frontend (mww_create_multi): every call runs the frontend once per stream tile and
    each model on its rows, and the staged host / peer paths copy the audio once.  `models`: a list of paths to (or bytes
    of) MWW containers or streaming ``.tflite`` flatbuffers, converted as StreamEngine converts them; any mix of kinds,
    geometries and strides.  Calls return one result per model, in the order of `models`; model k's results and state are
    bit-identical to a StreamEngine of models[k] given the same calls.  `stride`, `is_quantized`, `state_elements` and
    `pending_rows` are per-model lists.

    `streams`: None (every model on every stream) or one entry per model, None (all streams) or a strictly increasing
    sequence of stream ids (mww_create_multi_streams): model k then runs on those streams only, its state is allocated for
    them only, and its results have one row per id, in that order (row j belongs to stream streams[k][j]).  Unsorted,
    duplicate or out-of-range ids raise ValueError.  `engine.streams[k]` is model k's set (int32), `set_streams` changes it."""

    def __init__(self, models, n_streams: int = 1, device: int = 0, streams=None, input_rate: int = 16000, stream_rates=None,
                 stream_formats=None):
        if stream_rates is not None and input_rate != 16000:
            raise ValueError("give input_rate= or stream_rates=, not both")
        if stream_formats is not None and stream_rates is None:
            raise ValueError("stream_formats= needs stream_rates= (sample formats per stream need per-stream rates)")
        blobs = [load_model_blob(m) for m in models]
        if any(b is None for b in blobs):
            raise ValueError("every model must be a path or the bytes of a model file")
        K = len(blobs)
        if streams is not None and len(streams) != K:
            raise ValueError("streams must hold one entry per model (%d), not %d" % (K, len(streams)))
        sets = [None if streams is None or streams[k] is None else self._stream_set(streams[k], n_streams) for k in range(K)]
        self._L = _lib.lib()
        self._h = ctypes.c_void_p()
        self._bufs = [ctypes.create_string_buffer(b, len(b)) for b in blobs]
        ptrs = (ctypes.c_void_p * max(K, 1))(*[ctypes.addressof(b) for b in self._bufs])
        sizes = (ctypes.c_size_t * max(K, 1))(*[len(b) for b in blobs])
        if any(s is not None for s in sets):
            ids = (ctypes.c_void_p * K)(*[None if s is None else s.ctypes.data for s in sets])
            n_ids = (ctypes.c_int * K)(*[0 if s is None else s.size for s in sets])
            rc = self._L.mww_create_multi_streams(ptrs, sizes, K, int(device), int(n_streams), ids, n_ids, ctypes.byref(self._h))
        else:
            rc = self._L.mww_create_multi(ptrs, sizes, K, int(device), int(n_streams), ctypes.byref(self._h))
        if rc != 0:
            msg = self._L.mww_last_error(None)
            raise _lib.MwwError(rc, msg.decode() if msg else "mww_create_multi failed")
        self._bufs = None
        self.n_streams = int(n_streams)
        self.device = int(device)
        self.n_models = K
        infos = [self._model_info(k) for k in range(K)]
        self.is_quantized = [bool(i.is_quantized) for i in infos]
        self.stride = [max(int(i.input_feature_slices), 1) for i in infos]
        self.state_elements = [int(i.state_bytes_per_stream) // (1 if q else 4) for i, q in zip(infos, self.is_quantized)]
        self.hop = HOP
        self.streams = [self._get_streams(k) for k in range(K)]
        if input_rate != 16000:
            self.set_input_rate(input_rate)
        if stream_rates is not None:
            self.set_stream_rates(np.arange(self.n_streams, dtype=np.int32), stream_rates)
        if stream_formats is not None:
            self.set_stream_formats(np.arange(self.n_streams, dtype=np.int32), stream_formats)

    @staticmethod
    def _stream_set(ids, n_streams: int) -> np.ndarray:
        """a caller's stream ids -> int32 array; ValueError unless strictly increasing in [0, n_streams) (never sorted here:
        row j of a model's results belongs to its j-th id)"""
        a = np.asarray(ids)
        if a.ndim != 1 or (a.size and not np.issubdtype(a.dtype, np.integer)):
            raise ValueError("stream ids must be a 1-D sequence of integers")
        a = a.astype(np.int64)
        if a.size and (a[0] < 0 or a[-1] >= n_streams or (a.size > 1 and not (np.diff(a) > 0).all())):
            raise ValueError("stream ids must be strictly increasing and in [0, n_streams=%d)" % n_streams)
        return np.ascontiguousarray(a, np.int32)

    def _get_streams(self, k: int) -> np.ndarray:
        out = np.zeros(self.n_streams, np.int32)
        n = ctypes.c_int(0)
        _lib.check(self._h, self._L.mww_get_model_streams(self._h, int(k), out.ctypes.data, out.size, ctypes.byref(n)))
        return out[:n.value].copy()

    def set_streams(self, k: int, ids) -> None:
        """Model k runs on stream ids `ids` from now on (None: all streams), ordered on the current CUDA stream
        (mww_set_model_streams): streams it keeps continue exactly, streams that join start from fresh state."""
        if not 0 <= int(k) < self.n_models:
            raise ValueError("model index out of range")
        s = None if ids is None else self._stream_set(ids, self.n_streams)
        _lib.check(self._h, self._L.mww_set_model_streams(self._h, int(k), None if s is None else s.ctypes.data,
                                                          0 if s is None else s.size, self._cu_stream()))
        self.streams[int(k)] = self._get_streams(k)

    def _model_info(self, k: int):
        info = _lib.MwwInfo()
        _lib.check(self._h, self._L.mww_get_model_info(self._h, int(k), ctypes.byref(info)))
        return info

    @property
    def pending_rows(self) -> list:
        return [self._model_info(k).pending_rows for k in range(self.n_models)]

    def _steps(self, n_samples: int) -> list:
        rate, seen = self._rate()
        return call_plan(self.frontend_buffered, n_samples, self.hop, self.pending_rows, self.stride, rate, seen)[1]

    def _outs(self, steps, out, host: bool):
        """-> (K buffers, their ctypes pointer / max_probs / steps-out arrays); model k's buffer has one row per stream of
        its set"""
        torch = _torch()
        rows = [s.size for s in self.streams]
        if out is None:
            out = [np.empty((r, max(s, 1)), np.float32) if host else
                   torch.empty((r, max(s, 1)), dtype=torch.float32, device=self._dev()) for r, s in zip(rows, steps)]
        elif len(out) != self.n_models:
            raise ValueError("out must hold one buffer per model (%d)" % self.n_models)
        elif host:
            if any(o.dtype != np.float32 or o.ndim != 2 or o.shape[0] != r or not o.flags.c_contiguous for o, r in zip(out, rows)):
                raise ValueError("out must be C-contiguous float32 host arrays [streams of model k, >= steps]")
        else:
            for o, r in zip(out, rows):
                if o.dtype != torch.float32 or not o.is_cuda or not o.is_contiguous() or o.dim() != 2 or o.shape[0] != r:
                    raise ValueError("out must be contiguous CUDA float32 tensors [streams of model k, >= steps]")
        K = self.n_models
        ptrs = (ctypes.c_void_p * K)(*[o.ctypes.data if host else o.data_ptr() for o in out])
        maxp = (ctypes.c_int * K)(*[o.shape[1] for o in out])
        return out, ptrs, maxp, (ctypes.c_int * K)()

    def predict_clip(self, audio, out=None, samples16=None, law=None, mixed=False) -> list:
        """int16 or float32 CUDA tensor [S, N] -> [float32 probabilities [S, steps_k] for each model k]; state carries over
        between calls.  `out`: one CUDA float32 buffer [S, >= steps_k] per model to write into.  samples16=, law= and
        mixed=: as StreamEngine.predict_clip."""
        width, stride, _ = self._check_audio(audio, law, mixed)
        n = self._mixed_len(width, max(stride, width), audio.data_ptr(), samples16) if mixed else self._call_len(width, samples16)
        out, ptrs, maxp, got = self._outs(self._steps(n), out, False)
        fn = self._audio_fn("mww_predict_clip_multi", _kind(audio.dtype), law, mixed)
        _lib.check(self._h, fn(self._h, audio.data_ptr(), n, max(stride, width), ptrs, maxp, got, self._cu_stream()))
        return [o[:, :g] for o, g in zip(out, got)]

    def step(self, audio, out=None, law=None, mixed=False) -> list:
        """predict_clip; with per-stream rates a 30 ms call (samples16 = 480)"""
        return self.predict_clip(audio, out, LIVE_SAMPLES16 if self.per_stream_rates else None, law=law, mixed=mixed)

    def predict_clip_host(self, audio: np.ndarray, out=None, samples16=None, law=None, mixed=False) -> list:
        """int16 or float32 HOST array (uint8 with law= or mixed=True) [S, N] -> [float32 HOST array [S, steps_k] for each
        model k]; each audio tile is copied once."""
        audio, stride, _ = self._check_host_audio(audio, law, mixed)
        n = self._mixed_len(audio.shape[1], stride, audio.ctypes.data, samples16) if mixed else self._call_len(audio.shape[1], samples16)
        out, ptrs, maxp, got = self._outs(self._steps(n), out, True)
        fn = self._audio_fn("mww_predict_clip_host_multi", _kind(audio.dtype), law, mixed)
        _lib.check(self._h, fn(self._h, audio.ctypes.data, n, stride, ptrs, maxp, got))
        return [o[:, :g] for o, g in zip(out, got)]

    def predict_clip_remote(self, src_ptr: int, n_samples: int, stride: int | None = None, tiles: int = 0, out=None,
                            dtype=None, samples16=None, law=None, mixed=False) -> list:
        """StreamEngine.predict_clip_remote for every model: one result per model, each audio tile pulled once."""
        fn = self._remote_fn(dtype, "mww_predict_clip_remote_multi", law, mixed)
        width = int(n_samples)
        n = self._mixed_len(width, int(stride) if stride else width, int(src_ptr), samples16) if mixed else self._call_len(width, samples16)
        out, ptrs, maxp, got = self._outs(self._steps(n), out, False)
        _lib.check(self._h, fn(self._h, ctypes.c_void_p(int(src_ptr)), n, int(stride) if stride else width, ptrs, maxp, got, int(tiles),
                               self._cu_stream()))
        return [o[:, :g] for o, g in zip(out, got)]

    # ------------------------------------------------------------------ state (checkpoint / tests)
    def state_dict(self) -> dict:
        """{carry, estimate, frontend_buffered: the shared frontend; models: [{streams, nn, pending, pending_rows} per model]},
        model k's nn / pending arrays one row per stream of its set"""
        S = self.n_streams
        d = dict(carry=np.zeros((S, WINDOW), np.int16), estimate=np.zeros((S, NUM_FEATURES), np.uint32))
        _lib.check(self._h, self._L.mww_get_state(self._h, d["carry"].ctypes.data, d["estimate"].ctypes.data, None, None))
        d["frontend_buffered"] = self._info().frontend_buffered
        d["models"] = []
        for k in range(self.n_models):
            dt = np.int8 if self.is_quantized[k] else np.float32
            M = self.streams[k].size
            m = dict(streams=self.streams[k].copy(), nn=np.zeros((M, self.state_elements[k]), dt),
                     pending=np.zeros((M, max(self.stride[k] - 1, 1), NUM_FEATURES), dt))
            _lib.check(self._h, self._L.mww_get_model_state(self._h, k, m["nn"].ctypes.data, m["pending"].ctypes.data))
            m["pending_rows"] = self._model_info(k).pending_rows
            d["models"].append(m)
        self._get_resampler(d)
        return d

    def load_state_dict(self, d: dict) -> None:
        """the state of state_dict(); each model's stream set is restored first (a state without `streams`: all streams)"""
        if len(d["models"]) != self.n_models:
            raise ValueError("the state holds %d models, this engine %d" % (len(d["models"]), self.n_models))
        self._set_resampler(d)
        carry = np.ascontiguousarray(d["carry"], np.int16)
        est = np.ascontiguousarray(d["estimate"], np.uint32)
        for k, m in enumerate(d["models"]):
            want = self._stream_set(m["streams"], self.n_streams) if m.get("streams") is not None else np.arange(self.n_streams, dtype=np.int32)
            if not np.array_equal(want, self.streams[k]):
                self.set_streams(k, want)
        _lib.check(self._h, self._L.mww_set_state(self._h, carry.ctypes.data, int(d["frontend_buffered"]), est.ctypes.data, None, None, 0))
        for k, m in enumerate(d["models"]):
            dt = np.int8 if self.is_quantized[k] else np.float32
            nn = np.ascontiguousarray(m["nn"], dt)
            pend = np.ascontiguousarray(m["pending"], dt)
            M = self.streams[k].size
            if nn.shape != (M, self.state_elements[k]) or pend.shape != (M, max(self.stride[k] - 1, 1), NUM_FEATURES):
                raise ValueError("model %d: nn / pending must have one row per stream of its set (%d)" % (k, M))
            _lib.check(self._h, self._L.mww_set_model_state(self._h, k, nn.ctypes.data, pend.ctypes.data, int(m["pending_rows"])))
