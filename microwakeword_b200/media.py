"""The media guard on the GPU (mww_media_guard_* and mww_media_* of include/mww.h): a TV advert, a podcast or a broadcast that
says the wake word makes many households fire within a second, and every one of those detections is a true positive for the
wake model and the verifier.  A broadcast is the same audio heard in many homes at once.  The guard fingerprints the clip of
every detection, compares it with the other households' recent detections and with registered media clips, and takes the
matches out of what gets armed:

    scores, confirmed = ver.verify(eng, det, at_event=True, post=3200)
    matches, media, passed = guard.check(eng, det, confirmed, post=3200)
    ep.arm(passed)

The fingerprint is the Haitsma-Kalker energy-difference sign over the frontend's own feature rows: 39 bits per 10 ms frame.
Two clips match when, at some lag, at most `max_ber` of the overlapping bits differ.
"""

from __future__ import annotations

import ctypes
import weakref

import numpy as np

from . import _lib
from .detection import EVENT_DTYPE, MODEL_EVENT_DTYPE, MultiModelDetector, _Detector, _record_ids
from .engine import MAX_AUDIO_HISTORY

SAMPLE_RATE = 16000


def _int(value, name: str) -> int:
    if isinstance(value, bool) or not isinstance(value, (int, np.integer)):
        raise ValueError("%s must be an integer (got %r)" % (name, value))
    return int(value)


def _num(value, name: str) -> float:
    if isinstance(value, bool) or not isinstance(value, (int, float, np.integer, np.floating)) or not np.isfinite(value):
        raise ValueError("%s must be a finite number (got %r)" % (name, value))
    return float(value)


def frames(n_samples: int) -> int:
    """T, the feature rows of a clip of n_samples on a fresh frontend"""
    return (n_samples - 480) // 160 + 1


class MediaGuard:
    """A media guard on `slots` slots (at least a detector's capacity) with a fixed rule (include/mww.h, "media guard"):

    - n_samples: the clip of each detection, [640, 160000] samples at 16 kHz (T = (n_samples - 480) / 160 + 1 frames,
      T - 1 fingerprint words);
    - max_lag: frames of jitter allowed between two households' detections of one broadcast, [0, 64];
    - min_overlap: fewest overlapping words of a match, by default (T - 1) - max_lag;
    - max_ber: the largest share of differing bits in a match, [0, 0.5], in thousandths;
    - min_matches: the other-household matches that flag a detection as broadcast;
    - ring: recent detections kept for later checks, [0, 2**20]; window_s: how far apart on the audio axis two detections
      may be and still be compared;
    - max_media / max_media_s: how many media clips register() takes, and how long each may be.

    The defaults (n_samples=24000, max_lag=15, max_ber=0.30, min_matches=3, ring=8192, window_s=60) are guesses that nobody
    has measured.  How often genuine wakes in different homes (different speakers saying the same phrase) match each other,
    and how well a broadcast survives real rooms, are not known: there is no real speech to measure them on.  The tests show
    only that the rule is implemented as stated, on synthetic audio.

    Calls on one guard are ordered on the current CUDA stream."""

    def __init__(self, slots: int, n_samples: int = 24000, max_lag: int = 15, min_overlap=None, max_ber: float = 0.30,
                 min_matches: int = 3, ring: int = 8192, window_s: float = 60, max_media: int = 16, max_media_s: float = 30,
                 device: int = 0):
        slots, n_samples, max_lag = _int(slots, "slots"), _int(n_samples, "n_samples"), _int(max_lag, "max_lag")
        min_matches, ring, max_media, device = _int(min_matches, "min_matches"), _int(ring, "ring"), _int(max_media, "max_media"), _int(device, "device")
        max_ber, window_s, max_media_s = _num(max_ber, "max_ber"), _num(window_s, "window_s"), _num(max_media_s, "max_media_s")
        if slots < 1:
            raise ValueError("slots must be at least 1 (got %d)" % slots)
        if not 640 <= n_samples <= 160000:
            raise ValueError("n_samples must be in [640, 160000] (got %d)" % n_samples)
        words = frames(n_samples) - 1
        if not 0 <= max_lag <= 64:
            raise ValueError("max_lag must be in [0, 64] (got %d)" % max_lag)
        min_overlap = words - max_lag if min_overlap is None else _int(min_overlap, "min_overlap")
        if not 1 <= min_overlap <= words or max_lag > words - min_overlap:
            raise ValueError("min_overlap must be in [1, %d] with max_lag <= %d - min_overlap (got %d)" % (words, words, min_overlap))
        if not 0 <= max_ber <= 0.5:
            raise ValueError("max_ber must be in [0, 0.5] (got %r)" % max_ber)
        if min_matches < 1:
            raise ValueError("min_matches must be at least 1 (got %d)" % min_matches)
        if not 0 <= ring <= 1 << 20:
            raise ValueError("ring must be in [0, 2**20] (got %d)" % ring)
        window = int(round(window_s * SAMPLE_RATE))
        if not 0 <= window <= 1 << 40:
            raise ValueError("window_s must give [0, 2**40] samples (got %r)" % window_s)
        if not 0 <= max_media <= 4096:
            raise ValueError("max_media must be in [0, 4096] (got %d)" % max_media)
        max_media_samples = int(round(max_media_s * SAMPLE_RATE)) if max_media else 0
        if max_media and not (640 <= max_media_samples <= 1 << 24 and frames(max_media_samples) - 1 >= min_overlap):
            raise ValueError("max_media_s must give [640, 2**24] samples and at least min_overlap words (got %r)" % max_media_s)
        self._L = _lib.lib()
        self.rule = _lib.MwwMediaRule(n_samples, max_lag, min_overlap, int(round(max_ber * 1000)), min_matches, ring, max_media,
                                      max_media_samples, window)
        g = ctypes.c_void_p()
        self._g = None
        self._check(self._L.mww_media_guard_create(device, slots, ctypes.byref(self.rule), ctypes.byref(g)))
        self._g = g.value
        self.slots, self.n_samples, self.device, self.words = slots, n_samples, device, words
        self._last = weakref.WeakKeyDictionary()   # detector -> (matches, media) of the last check(engine, detector)

    def _check(self, rc: int) -> None:
        if rc != 0:
            msg = self._L.mww_last_error(None)
            raise _lib.MwwError(rc, msg.decode() if msg else "media guard call failed")

    def info(self) -> "_lib.MwwMediaGuardDesc":
        """mww_media_guard_info: the rule, frames, registered clips, ring fill and launches; waits for the device"""
        out = _lib.MwwMediaGuardDesc()
        self._check(self._L.mww_media_guard_info(self._g, ctypes.byref(out)))
        return out

    @property
    def launch_count(self) -> int:
        return int(self.info().launches)

    def close(self) -> None:
        if getattr(self, "_g", None):
            self._L.mww_media_guard_destroy(self._g)
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

    def check(self, engine, det_or_ids, confirmed=None, model=None, post: int = 0, ends=None, households=None):
        """-> (matches, media, passed): CUDA int32 tensors, ordered on the current CUDA stream.
        With a timed detector: one result per event slot [capacity] (slot i is drained event i), the clip ending `post`
        samples after each event, households the events' groups (-1 on an ungrouped detector); `model` = k checks only
        model k's events of a MultiModelDetector.  With stream ids (a host sequence or a CUDA int32 tensor): `ends` [n]
        int64 clip ends on the history axis, and `households` [n] int32 or None (every stream its own household).
        `confirmed` [n] (e.g. Verifier.verify's) is what passes when a slot is not flagged; None passes the slot's stream."""
        import torch
        if getattr(engine, "device", None) != self.device:
            raise ValueError("the engine must be on cuda:%d, the guard's device" % self.device)
        if engine.audio_history_capacity < self.n_samples:
            raise ValueError("the engine keeps %d samples of audio history; the guard reads %d (set_audio_history)"
                             % (engine.audio_history_capacity, self.n_samples))
        dev = torch.device("cuda", self.device)
        if isinstance(det_or_ids, _Detector):
            det = det_or_ids
            if not det.timed:
                raise ValueError("the media guard needs a timed detector (timed=True): its events carry their positions")
            if ends is not None or households is not None:
                raise ValueError("ends and households come from the detector")
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
            if households is not None:
                households = self._device_vector(households, torch.int32, n, "households")
        if confirmed is not None:
            confirmed = self._device_vector(confirmed, torch.int32, n, "confirmed")
        st = self._stream()
        matches, media, passed = (torch.empty(n, dtype=torch.int32, device=dev) for _ in range(3))
        cptr = confirmed.data_ptr() if confirmed is not None else None
        if isinstance(det_or_ids, _Detector):
            k = -1 if model is None else int(model)
            self._check(self._L.mww_media_check_detections_at(self._g, engine._h, det._d, k, post, cptr, matches.data_ptr(),
                                                              media.data_ptr(), passed.data_ptr(), st))
            self._last[det] = (matches, media)
        else:
            self._check(self._L.mww_media_check_streams(self._g, engine._h, ids.data_ptr(), ends.data_ptr(),
                                                        households.data_ptr() if households is not None else None, n, cptr,
                                                        matches.data_ptr(), media.data_ptr(), passed.data_ptr(), st))
        return matches, media, passed

    def register(self, clip) -> int:
        """Register a known media clip (an advert, a jingle): 16 kHz int16, or float32 in [-1, 1] converted as the frontend
        converts it, on the host or on CUDA, of at most max_media_s seconds.  Every later check flags (media bit 0) a
        detection whose clip matches it at any lag.  -> its index."""
        import torch
        dev = torch.device("cuda", self.device)
        x = clip if isinstance(clip, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(clip))
        if x.dim() != 1 or x.dtype not in (torch.int16, torch.float32):
            raise ValueError("a media clip is 1-D int16 or float32 audio at 16 kHz")
        n = x.numel()
        mx = self.rule.max_media_samples
        if self.rule.max_media == 0 or not 640 <= n <= mx or frames(n) - 1 < self.rule.min_overlap:
            raise ValueError("a media clip must have [640, %d] samples and at least min_overlap words (got %d)" % (mx, n))
        x = x.to(dev)
        if x.dtype == torch.float32:                 # mww_features_f32's rule: int16(trunc(clamp(x * 32768))), NaN -> 0
            x = torch.nan_to_num(x * 32768.0, nan=0.0).clamp(-32768.0, 32767.0).trunc().to(torch.int16)
        x = x.contiguous()
        idx = ctypes.c_int(0)
        self._check(self._L.mww_media_register(self._g, x.data_ptr(), n, ctypes.byref(idx), self._stream()))
        torch.cuda.current_stream(dev).synchronize()  # the clip's memory may go once register returns
        return idx.value

    def clear_registered(self) -> None:
        self._check(self._L.mww_media_clear_registered(self._g))

    def clear_ring(self) -> None:
        """forget every recent detection: after engine.set_audio_history, which restarts the audio axis"""
        self._check(self._L.mww_media_clear_ring(self._g))

    def state_dict(self) -> dict:
        """{"state": uint8 blob of the ring and the registered clips (include/mww.h layout)}; waits for the device"""
        n = ctypes.c_longlong(0)
        self._check(self._L.mww_media_get_state(self._g, None, ctypes.byref(n)))
        buf = np.zeros(n.value, np.uint8)
        self._check(self._L.mww_media_get_state(self._g, buf.ctypes.data, ctypes.byref(n)))
        return {"state": buf}

    def load_state_dict(self, d: dict) -> None:
        buf = np.ascontiguousarray(d["state"], np.uint8)
        self._check(self._L.mww_media_set_state(self._g, buf.ctypes.data, buf.size))

    def drain(self, detector, verifier=None):
        """detector.drain() with `matches` and `media` from the last check(engine, detector), paired by slot before the sort
        (-1 and 0 without one), and `verifier_score` when a verifier is given.  Waits for the current CUDA stream."""
        multi = isinstance(detector, MultiModelDetector)
        base, keys = (MODEL_EVENT_DTYPE, ("model", "step", "stream")) if multi else (EVENT_DTYPE, ("step", "stream"))
        ev, n = detector._drain_slots(base)
        last = self._last.pop(detector, None)
        extra = [("matches", np.int32), ("media", np.int32)] + ([("verifier_score", np.float32)] if verifier is not None else [])
        out = np.empty(ev.size, np.dtype(ev.dtype.descr + extra))
        for name in ev.dtype.names:
            out[name] = ev[name]
        out["matches"], out["media"] = (last[0][:ev.size].cpu().numpy(), last[1][:ev.size].cpu().numpy()) if last else (-1, 0)
        if verifier is not None:
            scores = verifier._last.pop(detector, None)
            out["verifier_score"] = scores[:ev.size].cpu().numpy() if scores is not None else np.nan
        return out[np.lexsort(tuple(out[k] for k in reversed(keys)))], max(n - detector.capacity, 0)
