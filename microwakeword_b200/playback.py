"""The playback guard on the GPU (mww_playback_* of include/mww.h): a satellite plays what the server sends it -- replies,
music -- and its microphone hears that playback.  A reply that says the wake word fires the stream, and for the wake model and
the verifier that is a true positive.  The server knows what it sent, so the guard keeps each stream's playback on the GPU, on
the engine's audio axis, and scores it at each detection with a wake model: a detection is suppressed when the device itself
said the wake word in the delay window before it.

    pb.play(ids, reply_audio)                                  # where replies are sent to the satellites
    ...
    scores, confirmed = ver.verify(eng, det, at_event=True, post=3200)
    _, _, passed = guard.check(eng, det, confirmed, post=3200)
    _, _, passed = pb.check(det, passed, post=3200)
    ep.arm(passed)

The rule never looks at the microphone audio: a user who says the wake word over music passes, and one who says it over the
device saying it is suppressed.
"""

from __future__ import annotations

import ctypes
import weakref

import numpy as np

from . import _lib
from .detection import EVENT_DTYPE, MODEL_EVENT_DTYPE, MultiModelDetector, _Detector, _record_ids
from .engine import MAX_AUDIO_HISTORY, WINDOW, load_model_blob

SAMPLE_RATE = 16000
MAX_START = 1 << 50


def _int(value, name: str) -> int:
    if isinstance(value, bool) or not isinstance(value, (int, np.integer)):
        raise ValueError("%s must be an integer (got %r)" % (name, value))
    return int(value)


def _num(value, name: str) -> float:
    if isinstance(value, bool) or not isinstance(value, (int, float, np.integer, np.floating)) or not np.isfinite(value):
        raise ValueError("%s must be a finite number (got %r)" % (name, value))
    return float(value)


def _pcm16(x, dev):
    """int16 audio on dev from int16, or float32 in [-1, 1] converted as the frontend converts it, on the host or on CUDA"""
    import torch
    x = x if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(x))
    if x.dtype not in (torch.int16, torch.float32):
        raise ValueError("playback audio is int16 or float32 at 16 kHz")
    x = x.to(dev)
    if x.dtype == torch.float32:                 # mww_features_f32's rule: int16(trunc(clamp(x * 32768))), NaN -> 0
        x = torch.nan_to_num(x * 32768.0, nan=0.0).clamp(-32768.0, 32767.0).trunc().to(torch.int16)
    return x


class PlaybackGuard:
    """A playback guard bound to `engine` (which must keep an audio history) with a wake model (`model`: what StreamEngine
    accepts) on `slots` slots (at least a detector's capacity), `rows` playback rows of `capacity_s` seconds, and a fixed rule
    (include/mww.h, "playback guard"):

    - n_samples: what the model must hear, at least 480 samples at 16 kHz;
    - min_delay, max_delay: the samples between a playback position and where the microphone hears it, 0 <= min_delay <=
      max_delay <= 2**22; the reference clip is the L_ref = n_samples + max_delay - min_delay samples that end min_delay before
      each clip end;
    - window, ignore_steps: the verifier's score over the reference clip; cutoff: a detection is flagged when that score is
      above it.

    capacity_s must cover the longest write made ahead of time plus L_ref.  The defaults (rows = min(n_streams, 4096), 10 s,
    n_samples=24000, delays 0..4800, window=5, ignore_steps=25, cutoff=0.5) are guesses that nobody has measured: how often real
    replies or music self-wake, and how often suppression costs a genuine barge-in, are not known.  The tests show only that
    the rule is implemented as stated, on synthetic audio.

    Calls on one guard are ordered on the current CUDA stream."""

    def __init__(self, model, engine, slots: int, rows=None, capacity_s: float = 10.0, n_samples: int = 24000, min_delay: int = 0,
                 max_delay: int = 4800, window: int = 5, ignore_steps: int = 25, cutoff: float = 0.5):
        slots, n_samples = _int(slots, "slots"), _int(n_samples, "n_samples")
        min_delay, max_delay = _int(min_delay, "min_delay"), _int(max_delay, "max_delay")
        window, ignore_steps, cutoff, capacity_s = _int(window, "window"), _int(ignore_steps, "ignore_steps"), _num(cutoff, "cutoff"), _num(capacity_s, "capacity_s")
        n_streams = engine.n_streams
        rows = min(n_streams, 4096) if rows is None else _int(rows, "rows")
        if slots < 1:
            raise ValueError("slots must be at least 1 (got %d)" % slots)
        if not 1 <= rows <= n_streams:
            raise ValueError("rows must be in [1, %d] (got %d)" % (n_streams, rows))
        capacity = int(round(capacity_s * SAMPLE_RATE / 8)) * 8
        if not 8 <= capacity <= MAX_AUDIO_HISTORY:
            raise ValueError("capacity_s must give [8, 2**22] samples (got %r)" % capacity_s)
        if n_samples < WINDOW:
            raise ValueError("n_samples must be at least %d (got %d)" % (WINDOW, n_samples))
        if not 0 <= min_delay <= max_delay <= MAX_AUDIO_HISTORY:
            raise ValueError("the delays must satisfy 0 <= min_delay <= max_delay <= 2**22 (got %d, %d)" % (min_delay, max_delay))
        l_ref = n_samples + max_delay - min_delay
        if l_ref > min(capacity, MAX_AUDIO_HISTORY):
            raise ValueError("n_samples + max_delay - min_delay = %d must be at most the capacity, %d samples" % (l_ref, capacity))
        if not 1 <= window <= 32:
            raise ValueError("window must be in [1, 32] (got %d)" % window)
        if ignore_steps < 0:
            raise ValueError("ignore_steps must not be negative (got %d)" % ignore_steps)
        if engine.audio_history_capacity == 0:
            raise ValueError("the engine keeps no audio history (set_audio_history): the guard uses its axis")
        blob = load_model_blob(model)
        if blob is None:
            raise ValueError("a playback guard needs a model, not a frontend-only engine")
        self._L = _lib.lib()
        self.rule = _lib.MwwPlaybackRule(n_samples, window, ignore_steps, 0, min_delay, max_delay, cutoff)
        g = ctypes.c_void_p()
        self._g = None
        self._check(self._L.mww_playback_guard_create(engine._h, blob, len(blob), slots, rows, capacity, ctypes.byref(self.rule), ctypes.byref(g)))
        self._g = g.value
        self.engine, self.device, self.n_streams = engine, engine.device, n_streams
        self.slots, self.rows, self.capacity, self.l_ref, self.cutoff = slots, rows, capacity, l_ref, cutoff
        self._last = weakref.WeakKeyDictionary()   # detector -> (scores, flagged) of the last check(detector)

    def _check(self, rc: int) -> None:
        if rc != 0:
            msg = self._L.mww_last_error(None)
            raise _lib.MwwError(rc, msg.decode() if msg else "playback guard call failed")

    def info(self) -> "_lib.MwwPlaybackGuardDesc":
        """mww_playback_guard_info: the rule, L_ref, steps, rows, rows_used, capacity and launches"""
        out = _lib.MwwPlaybackGuardDesc()
        self._check(self._L.mww_playback_guard_info(self._g, ctypes.byref(out)))
        return out

    @property
    def launch_count(self) -> int:
        return int(self.info().launches)

    def close(self) -> None:
        if getattr(self, "_g", None):
            self._L.mww_playback_guard_destroy(self._g)
            self._g = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _stream(self):
        import torch
        return ctypes.c_void_p(torch.cuda.current_stream(torch.device("cuda", self.device)).cuda_stream)

    def _device_vector(self, x, dtype, n, name):
        """x as a contiguous CUDA tensor [n] of dtype on the guard's device (host sequences are copied)"""
        import torch
        dev = torch.device("cuda", self.device)
        if isinstance(x, torch.Tensor) and x.is_cuda:
            if x.dtype != dtype or x.dim() != 1 or not x.is_contiguous() or x.device != dev or x.numel() != n:
                raise ValueError("%s must be a contiguous 1-D CUDA %s tensor of %d on %s" % (name, dtype, n, dev))
            return x
        a = np.asarray(x)
        if a.ndim != 1 or a.size != n or (a.size and not np.issubdtype(a.dtype, np.integer)):
            raise ValueError("%s must be %d integers" % (name, n))
        return torch.from_numpy(np.ascontiguousarray(a, {torch.int32: np.int32, torch.int64: np.int64}[dtype])).to(dev)

    def _ids(self, ids):
        ids = _record_ids(ids, "stream ids")
        if ids.size and (ids.min() < 0 or ids.max() >= self.n_streams):
            raise ValueError("stream ids must be in [0, %d)" % self.n_streams)
        return ids

    def play(self, ids, audio, starts=None) -> None:
        """Write playback: row i of `audio` [n, L] (int16, or float32 converted as the frontend converts it; host or CUDA) is
        what stream ids[i] plays from axis position starts[i].  starts=None puts each stream at max(its head,
        engine.audio_samples_seen), so a reply written in one go, or chunk by chunk, lands end to end from "now"."""
        ids = self._ids(ids)
        if len(set(ids.tolist())) != ids.size:
            raise ValueError("a stream id is listed twice")
        n = ids.size
        import torch
        x = _pcm16(audio, torch.device("cuda", self.device))
        if x.dim() == 1 and n == 1:
            x = x[None]
        if x.dim() != 2 or x.shape[0] != n:
            raise ValueError("audio must be [%d, samples]" % n)
        L = int(x.shape[1])
        if L > MAX_AUDIO_HISTORY:
            raise ValueError("a write is at most 2**22 samples per stream (got %d)" % L)
        if starts is None:
            _, heads = self.heads()
            starts = np.maximum(heads[ids], self.engine.audio_samples_seen)
        starts = np.ascontiguousarray(starts, np.int64)
        if starts.shape != (n,) or (n and np.abs(starts).max() > MAX_START):
            raise ValueError("starts must be %d positions in [-2**50, 2**50]" % n)
        x = x.contiguous()
        self._check(self._L.mww_playback_write(self._g, ids.ctypes.data, starts.ctypes.data, n, x.data_ptr() if n else None, L, L, self._stream()))

    def read(self, ids, ends, n: int):
        """-> CUDA int16 [len(ids), n]: each stream's playback over [end - n, end) (zeros where its row holds nothing)"""
        import torch
        n = _int(n, "n")
        if not 0 <= n <= MAX_AUDIO_HISTORY:
            raise ValueError("n must be in [0, 2**22] (got %d)" % n)
        ids = torch.from_numpy(self._ids(ids)) if not (isinstance(ids, torch.Tensor) and ids.is_cuda) else ids
        k = int(ids.numel())
        ids = self._device_vector(ids, torch.int32, k, "stream ids")
        ends = self._device_vector(ends, torch.int64, k, "ends")
        out = torch.zeros((k, n), dtype=torch.int16, device=torch.device("cuda", self.device))
        self._check(self._L.mww_playback_read(self._g, ids.data_ptr(), ends.data_ptr(), k, n, out.data_ptr(), n, self._stream()))
        return out

    def reset(self, ids=None) -> None:
        """free the rows of the listed streams (None: every stream; do that after engine.set_audio_history)"""
        if ids is None:
            self._check(self._L.mww_playback_reset(self._g, None, 0, self._stream()))
            return
        ids = self._ids(ids)
        self._check(self._L.mww_playback_reset(self._g, ids.ctypes.data, ids.size, self._stream()))

    def heads(self):
        """-> (rows, heads): int32 and int64 [n_streams], row -1 and head 0 for a stream without a row"""
        rows, heads = np.zeros(self.n_streams, np.int32), np.zeros(self.n_streams, np.int64)
        self._check(self._L.mww_playback_get_heads(self._g, rows.ctypes.data, heads.ctypes.data))
        return rows, heads

    def check(self, det_or_ids, confirmed=None, model=None, post: int = 0, ends=None):
        """-> (scores, flagged, passed): CUDA float32, int32 and int32 tensors, ordered on the current CUDA stream.
        With a timed detector: one result per event slot [capacity] (slot i is drained event i), the clip ending `post` samples
        after each event; `model` = k checks only model k's events of a MultiModelDetector.  With stream ids (a host sequence
        or a CUDA int32 tensor): `ends` [n] int64 clip ends on the audio axis.  `confirmed` [n] (e.g. MediaGuard.check's
        passed) is what passes when a slot is not flagged; None passes the slot's stream."""
        import torch
        dev = torch.device("cuda", self.device)
        if self.engine.audio_history_capacity == 0:
            raise ValueError("the engine keeps no audio history any more (set_audio_history)")
        if isinstance(det_or_ids, _Detector):
            det = det_or_ids
            if not det.timed:
                raise ValueError("the playback guard needs a timed detector (timed=True): its events carry their positions")
            if ends is not None:
                raise ValueError("ends come from the detector")
            if det.device != self.device:
                raise ValueError("the detector must be on cuda:%d, the guard's device" % self.device)
            if det.capacity > self.slots:
                raise ValueError("the detector keeps %d events; the guard has %d slots" % (det.capacity, self.slots))
            K = getattr(det, "n_models", 1)
            if model is not None and (isinstance(model, bool) or not isinstance(model, (int, np.integer)) or not 0 <= model < K):
                raise ValueError("model must be None or a model index in [0, %d) (got %r)" % (K, model))
            post = _int(post, "post")
            if not 0 <= post <= MAX_AUDIO_HISTORY:
                raise ValueError("post must be in [0, %d] (got %d)" % (MAX_AUDIO_HISTORY, post))
            n = det.capacity
        else:
            if model is not None or post != 0:
                raise ValueError("model and post apply to a detector; give stream ids their clip ends instead")
            ids = det_or_ids
            if not (isinstance(ids, torch.Tensor) and ids.is_cuda):
                ids = _record_ids(ids, "stream ids")
            n = int(ids.numel() if isinstance(ids, torch.Tensor) else ids.size)
            if n > self.slots:
                raise ValueError("%d stream ids for a guard of %d slots" % (n, self.slots))
            if ends is None:
                raise ValueError("stream ids need their clip ends (ends)")
            ids = self._device_vector(ids, torch.int32, n, "stream ids")
            ends = self._device_vector(ends, torch.int64, n, "ends")
        if confirmed is not None:
            confirmed = self._device_vector(confirmed, torch.int32, n, "confirmed")
        scores = torch.empty(n, dtype=torch.float32, device=dev)
        flagged, passed = (torch.empty(n, dtype=torch.int32, device=dev) for _ in range(2))
        cptr = confirmed.data_ptr() if confirmed is not None else None
        st = self._stream()
        if isinstance(det_or_ids, _Detector):
            k = -1 if model is None else int(model)
            self._check(self._L.mww_playback_check_detections_at(self._g, det._d, k, post, cptr, scores.data_ptr(), flagged.data_ptr(),
                                                                 passed.data_ptr(), st))
            self._last[det] = (scores, flagged)
        else:
            self._check(self._L.mww_playback_check_streams(self._g, ids.data_ptr(), ends.data_ptr(), n, cptr, scores.data_ptr(),
                                                           flagged.data_ptr(), passed.data_ptr(), st))
        return scores, flagged, passed

    def state_dict(self) -> dict:
        """{"ids": the playing streams, "heads": their heads, "audio": int16 [n, capacity], what each row holds, [head -
        capacity, head)}: a checkpoint, or a stream's playback moved to another guard (write at rebased starts)"""
        rows, heads = self.heads()
        ids = np.flatnonzero(rows >= 0).astype(np.int32)
        audio = self.read(ids, heads[ids], self.capacity).cpu().numpy() if ids.size else np.zeros((0, self.capacity), np.int16)
        return {"ids": ids, "heads": heads[ids], "audio": audio}

    def load_state_dict(self, d: dict) -> None:
        """every stream's playback as in `d`; streams not in it play nothing"""
        ids, heads = np.asarray(d["ids"], np.int32), np.asarray(d["heads"], np.int64)
        audio = np.asarray(d["audio"], np.int16)
        if audio.shape != (ids.size, self.capacity) or heads.shape != ids.shape:
            raise ValueError("the state is of a guard with another capacity, or malformed")
        self.reset()
        if ids.size:
            self.play(ids, audio, starts=heads - self.capacity)

    def drain(self, detector, verifier=None, media_guard=None):
        """detector.drain() with `playback_score` and `self_wake` from the last check(detector), paired by slot before the sort
        (NaN and 0 without one), `verifier_score` when a verifier is given and `matches` and `media` when a media guard is.
        Waits for the current CUDA stream."""
        multi = isinstance(detector, MultiModelDetector)
        base, keys = (MODEL_EVENT_DTYPE, ("model", "step", "stream")) if multi else (EVENT_DTYPE, ("step", "stream"))
        ev, n = detector._drain_slots(base)
        last = self._last.pop(detector, None)
        extra = [("playback_score", np.float32), ("self_wake", np.int32)]
        extra += [("verifier_score", np.float32)] if verifier is not None else []
        extra += [("matches", np.int32), ("media", np.int32)] if media_guard is not None else []
        out = np.empty(ev.size, np.dtype(ev.dtype.descr + extra))
        for name in ev.dtype.names:
            out[name] = ev[name]
        out["playback_score"], out["self_wake"] = (last[0][:ev.size].cpu().numpy(), last[1][:ev.size].cpu().numpy()) if last else (np.nan, 0)
        if verifier is not None:
            scores = verifier._last.pop(detector, None)
            out["verifier_score"] = scores[:ev.size].cpu().numpy() if scores is not None else np.nan
        if media_guard is not None:
            m = media_guard._last.pop(detector, None)
            out["matches"], out["media"] = (m[0][:ev.size].cpu().numpy(), m[1][:ev.size].cpu().numpy()) if m else (-1, 0)
        return out[np.lexsort(tuple(out[k] for k in reversed(keys)))], max(n - detector.capacity, 0)
