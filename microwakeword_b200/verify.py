"""Second-stage verification on the GPU (mww_verifier_* and mww_verify_* of include/mww.h): a second, usually larger model
re-scores the streams a detector just fired on, from the last `n_samples` of their audio history, and confirms the ones
whose score is above its cutoff.  The audio never leaves the GPU and the host is never synchronised:

    eng.set_audio_history(32000)
    ver = Verifier(big_model, slots=det.capacity, n_samples=32000, cutoff=0.9)
    det.update(eng.step(chunk))
    scores, confirmed = ver.verify(eng, det)       # before eng.reset: a reset zeroes the history
    eng.reset(confirmed)                           # restart only the confirmed streams
    events, dropped = ver.drain(det)               # now and then: events with their verifier_score

With a timed detector the clip can end at the event instead of "now" (at_event=True): the verifier then hears the same
n_samples around the wake word whatever the poll interval, post samples of them after the detection.

The score is the positive-sample score of the reference's streaming ROC (test.py:364-373): the verifier model on a fresh
frontend and fresh state over the clip, as the reference makes the spectrograms of its positive clips, then
detection.positive_scores with (window, ignore_steps).  So detection.streaming_model_roc picks a verifier cutoff by the rule
the verifier applies.
"""

from __future__ import annotations

import ctypes
import math
import weakref

import numpy as np

from . import _lib
from .detection import EVENT_DTYPE, MODEL_EVENT_DTYPE, MultiModelDetector, _Detector, _record_ids
from .engine import MAX_AUDIO_HISTORY, WINDOW, load_model_blob


def _int(value, name: str) -> int:
    if isinstance(value, bool) or not isinstance(value, (int, np.integer)):
        raise ValueError("%s must be an integer (got %r)" % (name, value))
    return int(value)


class Verifier:
    """One verifier model on `slots` scratch streams and a fixed rule: each verify reads the last `n_samples` 16 kHz samples
    of every listed stream's audio history (n_samples in [480, 2**22], at most the engine's history capacity), runs the model
    on them from fresh state, and scores the probabilities with the moving average of `window` (in [1, 32]) after
    `ignore_steps` probabilities.  A stream is confirmed when its score (as float64) is above `cutoff`.  `model`: what
    StreamEngine accepts (a container path or bytes, or a streaming .tflite; fp32, int8, any geometry, hybrid).

    By default the read is "now", not the samples that end at the event: a caller that verifies at each drain, every D live
    calls of 480 samples, needs n_samples to cover what the verifier must hear plus D * 480 samples.  verify(..., at_event=True)
    on a timed detector reads the clip that ends `post` samples after each event instead, so n_samples is only what the
    verifier hears.  Calls on one verifier are ordered on the current CUDA stream; the verifier's own model state is scratch."""

    def __init__(self, model, slots: int, n_samples: int, cutoff: float, window: int = 5, ignore_steps: int = 25, device: int = 0):
        slots, n_samples = _int(slots, "slots"), _int(n_samples, "n_samples")
        window, ignore_steps, device = _int(window, "window"), _int(ignore_steps, "ignore_steps"), _int(device, "device")
        if slots < 1:
            raise ValueError("slots must be at least 1 (got %d)" % slots)
        if not WINDOW <= n_samples <= MAX_AUDIO_HISTORY:
            raise ValueError("n_samples must be in [%d, %d] (got %d)" % (WINDOW, MAX_AUDIO_HISTORY, n_samples))
        if not 1 <= window <= 32:
            raise ValueError("window must be in [1, 32] (got %d)" % window)
        if ignore_steps < 0:
            raise ValueError("ignore_steps must not be negative (got %d)" % ignore_steps)
        if isinstance(cutoff, bool) or not isinstance(cutoff, (int, float, np.integer, np.floating)) or not math.isfinite(cutoff):
            raise ValueError("cutoff must be a finite number (got %r)" % (cutoff,))
        blob = load_model_blob(model)
        if blob is None:
            raise ValueError("a verifier needs a model, not a frontend-only engine")
        self._L = _lib.lib()
        rule = _lib.MwwVerifyRule(n_samples, window, ignore_steps, 0, float(cutoff))
        v = ctypes.c_void_p()
        self._v = None
        self._check(self._L.mww_verifier_create(blob, len(blob), device, slots, ctypes.byref(rule), ctypes.byref(v)))
        self._v = v.value
        desc = self._desc()
        self.slots, self.n_samples, self.window, self.ignore_steps = slots, n_samples, window, ignore_steps
        self.cutoff, self.device, self.steps = float(cutoff), device, int(desc.steps)
        self._last = weakref.WeakKeyDictionary()        # detector -> scores of its slots from the last verify(engine, detector)

    def _check(self, rc: int) -> None:
        if rc != 0:
            msg = self._L.mww_last_error(None)
            raise _lib.MwwError(rc, msg.decode() if msg else "verifier call failed")

    def _desc(self) -> "_lib.MwwVerifierDesc":
        out = _lib.MwwVerifierDesc()
        self._check(self._L.mww_verifier_info(self._v, ctypes.byref(out)))
        return out

    @property
    def launch_count(self) -> int:
        """kernel launches of the verifier's model handle since create: the same for every verify call"""
        return int(self._desc().launches)

    def close(self) -> None:
        if getattr(self, "_v", None):
            self._L.mww_verifier_destroy(self._v)
            self._v = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def verify(self, engine, ids_or_detector, model=None, at_event: bool = False, post: int = 0):
        """-> (scores, confirmed): CUDA float32 and int32 tensors, ordered on the current CUDA stream.
        `ids_or_detector`: stream ids of `engine` (a host sequence, or a contiguous 1-D CUDA int32 tensor such as a
        StreamDetector's fired_ids, whose -1 slots give NaN / -1), one result per id; or a detector, one result per event
        slot [capacity] (slot i is drained event i), with `model` = k verifying only model k's events of a
        MultiModelDetector.  An id outside [0, n_streams) scores NaN; confirmed[i] is the id or -1.
        `at_event=True` (a timed detector only): each slot's clip is the n_samples that end at e = min(sample + post,
        audio_samples_seen), `post` in [0, 2**22] samples after the event (mww_verify_detections_at).  An event younger than
        `post` is heard with a shorter post-roll; a slot whose clip has left the history ring scores NaN / -1."""
        import torch
        if at_event:
            if not isinstance(ids_or_detector, _Detector) or not ids_or_detector.timed:
                raise ValueError("at_event=True needs a timed detector (timed=True): its events carry their positions")
            post = _int(post, "post")
            if not 0 <= post <= MAX_AUDIO_HISTORY:
                raise ValueError("post must be in [0, %d] (got %d)" % (MAX_AUDIO_HISTORY, post))
        elif post != 0:
            raise ValueError("post applies to verify(..., at_event=True) only")
        dev = torch.device("cuda", self.device)
        if getattr(engine, "device", None) != self.device:
            raise ValueError("the engine must be on cuda:%d, the verifier's device" % self.device)
        if engine.audio_history_capacity < self.n_samples:
            raise ValueError("the engine keeps %d samples of audio history; the verifier reads %d (set_audio_history)"
                             % (engine.audio_history_capacity, self.n_samples))
        if isinstance(ids_or_detector, _Detector):
            det = ids_or_detector
            if det.device != self.device:
                raise ValueError("the detector must be on cuda:%d, the verifier's device" % self.device)
            if det.capacity > self.slots:
                raise ValueError("the detector keeps %d events; the verifier has %d slots" % (det.capacity, self.slots))
            K = getattr(det, "n_models", 1)
            if model is not None and (isinstance(model, bool) or not isinstance(model, (int, np.integer)) or not 0 <= model < K):
                raise ValueError("model must be None or a model index in [0, %d) (got %r)" % (K, model))
            n = det.capacity
        else:
            if model is not None:
                raise ValueError("model selects a detector's events; it has no meaning for a list of stream ids")
            ids = ids_or_detector
            if isinstance(ids, torch.Tensor) and ids.is_cuda:
                if ids.dtype != torch.int32 or ids.dim() != 1 or not ids.is_contiguous() or ids.device != dev:
                    raise ValueError("device stream ids must be a contiguous 1-D CUDA int32 tensor on %s" % dev)
            else:
                ids = torch.from_numpy(_record_ids(ids, "stream ids"))
            n = ids.numel()
            if n > self.slots:
                raise ValueError("%d stream ids for a verifier of %d slots" % (n, self.slots))
            ids = ids.to(dev)
        st = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        scores = torch.empty(n, dtype=torch.float32, device=dev)
        confirmed = torch.empty(n, dtype=torch.int32, device=dev)
        if isinstance(ids_or_detector, _Detector):
            k = -1 if model is None else int(model)
            if at_event:
                self._check(self._L.mww_verify_detections_at(self._v, engine._h, det._d, k, post, scores.data_ptr(), confirmed.data_ptr(), st))
            else:
                self._check(self._L.mww_verify_detections(self._v, engine._h, det._d, k, scores.data_ptr(), confirmed.data_ptr(), st))
            self._last[det] = scores
        else:
            self._check(self._L.mww_verify_streams(self._v, engine._h, ids.data_ptr(), n, scores.data_ptr(), confirmed.data_ptr(), st))
        return scores, confirmed

    def drain(self, detector):
        """detector.drain() with one more field, `verifier_score`: each event's score from the last verify(engine, detector)
        since the detector's last drain through this verifier, paired by slot; NaN for an event that fired after that verify,
        for another model's event, and when there was none.  A timed detector's events keep their `sample`.  Waits for the
        current CUDA stream, and clears the detector's events and fired_ids as its drain does."""
        multi = isinstance(detector, MultiModelDetector)
        base, keys = (MODEL_EVENT_DTYPE, ("model", "step", "stream")) if multi else (EVENT_DTYPE, ("step", "stream"))
        ev, n = detector._drain_slots(base)
        scores = self._last.pop(detector, None)
        out = np.empty(ev.size, np.dtype(ev.dtype.descr + [("verifier_score", np.float32)]))
        for name in ev.dtype.names:
            out[name] = ev[name]
        out["verifier_score"] = scores[:ev.size].cpu().numpy() if scores is not None else np.nan
        return out[np.lexsort(tuple(out[k] for k in reversed(keys)))], max(n - detector.capacity, 0)
