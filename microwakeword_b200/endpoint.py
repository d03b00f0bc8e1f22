"""Endpointing on the GPU (mww_endpointer_* of include/mww.h): after a wake word, find where each stream's spoken command
ends from a VAD model's probabilities, and cut the command's clip from the engine's audio history.  Nothing leaves the GPU
until the clips are wanted:

    eng.set_audio_history(16000 * 12)
    ep = Endpointer(eng, model=vad)                      # vad: the model index whose probabilities mean speech
    probs = eng.step(chunk)
    det.update(probs); ep.update(probs[vad])
    scores, confirmed = ver.verify(eng, det)
    ep.arm(confirmed)                                    # replays the last lookback_steps, so the command's start is kept
    ep.arm(passed, at=det)                               # or: start at each detection's position, after the wake word
    ...
    clips, lengths = ep.commands(pre=1600, post=3200, max_samples=16000 * 10)     # before the drain and the reset
    eng.reset(ep.ended_ids); det.reset(ep.ended_ids)
    events, dropped = ep.drain()

Every position is a sample index on the audio history's axis (engine.audio_samples_seen).  Steps are model steps: 30 ms at
stride 3 and a 10 ms hop, which is what the defaults are written for.
"""

from __future__ import annotations

import ctypes
import math

import numpy as np

from . import _lib
from .detection import _DeviceArray, _DetectorHandle, _record_ids
from .engine import MAX_AUDIO_HISTORY

MAX_SKIP = 1 << 22
MUTE_PLACED = 1 << 30              # the mute word's bit of a row armed at a position that has taken no step since

END_OF_SPEECH, NO_SPEECH, MAX_LENGTH = _lib.MWW_ENDPOINT_END_OF_SPEECH, _lib.MWW_ENDPOINT_NO_SPEECH, _lib.MWW_ENDPOINT_MAX_LENGTH
ENDPOINT_EVENT_DTYPE = np.dtype([("stream", np.int32), ("reason", np.int32), ("start_sample", np.int64), ("end_sample", np.int64),
                                 ("speech_end_sample", np.int64), ("steps", np.int32), ("pad", np.int32)])


def _int(value, name: str) -> int:
    if isinstance(value, bool) or not isinstance(value, (int, np.integer)):
        raise ValueError("%s must be an integer (got %r)" % (name, value))
    return int(value)


class EndpointerRecords:
    """Endpointer rows exported from an Endpointer (export_streams): `data`, torch.uint8 [n, record_bytes] on the
    endpointer's device, one packed record per listed stream (include/mww.h, "moving endpointer rows"), and `layout`, the
    _lib.MwwEndpointerLayout an importing endpointer must share.  Positions travel as ages from the exporter's baseline, so
    they land on the importer's axis.  The records carry no events.  layout.pad is 1 when the exporter was positioned
    (its records carry each armed row's mute word) and 0 otherwise."""

    _FIELDS = ("record_bytes", "vad_window", "stride", "hop_samples", "buffered", "pending", "pad", "samples_seen", "steps")

    def __init__(self, data, layout):
        self.data, self.layout = data, layout

    def save(self, path) -> None:
        """np.savez of the records and the layout's fields: a checkpoint of some streams' endpointer rows"""
        np.savez(path, data=self.data.cpu().numpy(), **{k: np.asarray(getattr(self.layout, k)) for k in self._FIELDS})

    @classmethod
    def load(cls, path, device) -> "EndpointerRecords":
        import torch
        layout = _lib.MwwEndpointerLayout()
        with np.load(path) as z:
            for k in cls._FIELDS:
                setattr(layout, k, int(z[k]))
            data = torch.from_numpy(z["data"]).to(device)
        return cls(data, layout)


class _EndpointerHandle(_DetectorHandle):
    """owner of one mww_endpointer_t: destroyed when the endpointer and every tensor over its buffers are gone"""

    def close(self):
        if self.ptr:
            self.L.mww_endpointer_destroy(self.ptr)
            self.ptr = None


class Endpointer:
    """Per-stream VAD endpointing of model `model` (None: 0) of `engine`, a StreamEngine or MultiModelEngine that keeps an
    audio history.  Each member stream of the model's stream set has a row.  Every row runs the models detector's VAD rule
    (moving average of `vad_window` probabilities above `vad_cutoff`) on every step; an armed row also runs the segmenter
    and ends with one event:

    - END_OF_SPEECH once speech was heard (`speech_steps` speech flags in a row; default 3 steps = 90 ms at 30 ms steps)
      and then `silence_steps` steps without speech (default 25 = 0.75 s);
    - NO_SPEECH when nothing was heard within `timeout_steps` (default 100 = 3 s);
    - MAX_LENGTH after `max_steps` (default 334, about 10 s).

    `lookback_steps` (0 .. 64, default 64 = 1.92 s) are replayed at arm, so arming late by the detector -> verifier
    latency changes nothing.  The replay reaches back over the wake word itself, which the VAD hears as speech: the segment
    (and the clip) starts before the wake word, and if the speaker pauses longer than `silence_steps` after it, the command
    ends with END_OF_SPEECH before it is spoken.  Set lookback_steps to the latency to cover, not more, and silence_steps
    above the pause speakers make after the wake word -- or arm at the detection's position, arm(ids, at=det), which starts
    the command after the wake word.  A whole reset() forgets the steps before it: no replay crosses it.
    `capacity` events are kept between drains; more are counted and dropped."""

    def __init__(self, engine, model=None, vad_window: int = 5, vad_cutoff: float = 0.5, speech_steps: int = 3, silence_steps: int = 25,
                 timeout_steps: int = 100, max_steps: int = 334, lookback_steps: int = 64, capacity: int = 4096):
        model = 0 if model is None else _int(model, "model")
        vad_window, capacity = _int(vad_window, "vad_window"), _int(capacity, "capacity")
        steps = {k: _int(v, k) for k, v in (("speech_steps", speech_steps), ("silence_steps", silence_steps),
                                            ("timeout_steps", timeout_steps), ("max_steps", max_steps))}
        lookback_steps = _int(lookback_steps, "lookback_steps")
        if not 1 <= vad_window <= 32:
            raise ValueError("vad_window must be in [1, 32] (got %d)" % vad_window)
        if isinstance(vad_cutoff, bool) or not isinstance(vad_cutoff, (int, float, np.integer, np.floating)) or not math.isfinite(vad_cutoff):
            raise ValueError("vad_cutoff must be a finite number (got %r)" % (vad_cutoff,))
        for k, v in steps.items():
            if v < 1:
                raise ValueError("%s must be at least 1 (got %d)" % (k, v))
        if not 0 <= lookback_steps <= 64:
            raise ValueError("lookback_steps must be in [0, 64] (got %d)" % lookback_steps)
        if capacity < 1:
            raise ValueError("capacity must be at least 1 (got %d)" % capacity)
        if getattr(engine, "_h", None) is None:
            raise ValueError("engine must be a StreamEngine or MultiModelEngine")
        if engine.audio_history_capacity == 0:
            raise ValueError("the engine keeps no audio history (set_audio_history)")
        n_models = getattr(engine, "n_models", 1)
        if not 0 <= model < n_models:
            raise ValueError("model must be in [0, %d) (got %d)" % (n_models, model))
        self._L = _lib.lib()
        rule = _lib.MwwEndpointRule(vad_window, steps["speech_steps"], steps["silence_steps"], steps["timeout_steps"], steps["max_steps"],
                                    lookback_steps, float(vad_cutoff))
        ep = ctypes.c_void_p()
        self._check(self._L.mww_endpointer_create(engine._h, model, ctypes.byref(rule), capacity, ctypes.byref(ep)))
        self._handle = _EndpointerHandle(self._L, ep.value)
        self.engine, self.model, self.device, self.capacity = engine, model, int(engine.device), capacity
        self.vad_window, self.vad_cutoff, self.lookback_steps = vad_window, float(vad_cutoff), lookback_steps
        self.speech_steps, self.silence_steps = steps["speech_steps"], steps["silence_steps"]
        self.timeout_steps, self.max_steps = steps["timeout_steps"], steps["max_steps"]
        desc = self._desc()
        self.n_rows, self.stride, self.hop = int(desc.n_rows), int(desc.stride), int(desc.hop_samples)
        count, ended, armed = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_void_p()
        self._check(self._L.mww_endpointer_buffers(self._ep, ctypes.byref(count), None, ctypes.byref(ended), ctypes.byref(armed), None))
        import torch
        dev = torch.device("cuda", self.device)
        with torch.cuda.device(dev):
            # device views: the stream of each used event slot (-1 elsewhere), every row's stream while armed (-1 elsewhere),
            # and how many commands ended since the last drain
            self.ended_ids = torch.as_tensor(_DeviceArray(self._handle, ended.value, capacity, "<i4"), device=dev)
            self.armed_ids = torch.as_tensor(_DeviceArray(self._handle, armed.value, max(self.n_rows, 1), "<i4"), device=dev)[:self.n_rows]
            self.event_count = torch.as_tensor(_DeviceArray(self._handle, count.value, 1, "<i8"), device=dev)

    @property
    def _ep(self):
        return self._handle.ptr

    def _check(self, rc: int) -> None:
        if rc != 0:
            msg = self._L.mww_last_error(None)
            raise _lib.MwwError(rc, msg.decode() if msg else "endpointer call failed")

    def _desc(self) -> "_lib.MwwEndpointerDesc":
        out = _lib.MwwEndpointerDesc()
        self._check(self._L.mww_endpointer_info(self._ep, ctypes.byref(out)))
        return out

    @property
    def launch_count(self) -> int:
        """kernel launches of this endpointer since create: one per update, arm, disarm, reset and commands call"""
        return int(self._desc().launches)

    def _stream(self):
        import torch
        return ctypes.c_void_p(torch.cuda.current_stream(torch.device("cuda", self.device)).cuda_stream)

    def close(self) -> None:
        """free the endpointer now; armed_ids, ended_ids and event_count must not be used afterwards"""
        self._handle.close()

    def update(self, probs) -> None:
        """The model's probabilities of the engine call just made: a StreamEngine result, or probs[model] of a MultiModelEngine
        result (CUDA float32 [n_rows, steps], any row pitch).  Call it after every engine call, steps or none: the endpointer
        places the steps on the history axis from the engine's counters and refuses an update that does not match them.
        Asynchronous on the current CUDA stream."""
        import torch
        if (not isinstance(probs, torch.Tensor) or not probs.is_cuda or probs.dtype != torch.float32 or probs.dim() != 2
                or probs.shape[0] != self.n_rows or probs.device.index != self.device):
            raise ValueError("probs must be a CUDA float32 tensor [n_rows=%d, steps] on cuda:%d" % (self.n_rows, self.device))
        n = probs.shape[1]
        if n and ((n > 1 and probs.stride(1) != 1) or (self.n_rows > 1 and probs.stride(0) < n)):
            probs = probs.contiguous()
        pitch = probs.stride(0) if self.n_rows > 1 else n
        self._check(self._L.mww_endpointer_update(self._ep, probs.data_ptr() if n and self.n_rows else None, n, pitch, self._stream()))

    def _ids_call(self, ids, host_fn: str, device_fn, allow_all: bool = False) -> None:
        """the host call `host_fn` or the device call `device_fn` (names; None: host ids only) on a checked id list"""
        import torch
        if ids is None and allow_all:
            self._check(getattr(self._L, host_fn)(self._ep, None, 0, self._stream()))
        elif isinstance(ids, torch.Tensor) and ids.is_cuda:
            if device_fn is None:
                raise ValueError("this call takes host stream ids")
            if ids.dtype != torch.int32 or ids.dim() != 1 or not ids.is_contiguous() or ids.device.index != self.device:
                raise ValueError("device stream ids must be a contiguous 1-D CUDA int32 tensor on cuda:%d" % self.device)
            self._check(getattr(self._L, device_fn)(self._ep, ids.data_ptr(), ids.numel(), self._stream()))
        else:
            a = _record_ids(ids, "stream ids")
            if a.size and (a.min() < 0 or a.max() >= self.engine.n_streams):
                raise ValueError("stream ids must be in [0, %d)" % self.engine.n_streams)
            self._check(getattr(self._L, host_fn)(self._ep, a.ctypes.data, a.size, self._stream()))

    def arm(self, ids, at=None, skip=None) -> None:
        """Start a command on the listed GLOBAL stream ids: a host sequence, or a contiguous 1-D CUDA int32 tensor such as a
        verifier's confirmed ids or a detector's fired_ids, whose -1 slots (and ids outside the model's stream set) are
        ignored.  Re-arming restarts a row; the last lookback_steps flags are replayed.

        at: each id's position on the audio history's axis (include/mww.h, "positioned arm"): the command starts there, not
        lookback_steps before the arm, so it leaves the wake word out.  It is one of
          - a timed StreamDetector or MultiModelDetector of this engine and device: its event_samples, slot for slot with
            ids, which must then be a CUDA int32 tensor of its capacity (passed, confirmed or fired_ids);
          - a CUDA int64 tensor beside CUDA ids;
          - a host sequence beside host ids.
        The steps within `skip` samples after a position take no speech (default vad_window * stride * hop, which covers the
        VAD average's lag behind the end of the wake word; a guess, not measured on real speech), so the wake word's tail
        does not count as the command.  A stream listed twice arms at its latest position.  The first positioned arm makes
        the endpointer positioned for good: every later call runs the positioned kernels, which give the same results while
        no row is muted."""
        if at is None:
            if skip is not None:
                raise ValueError("skip applies to a positioned arm (at=...)")
            self._ids_call(ids, "mww_endpointer_arm", "mww_endpointer_arm_device")
            return
        skip = self.vad_window * self.stride * self.hop if skip is None else _int(skip, "skip")
        if not 0 <= skip <= MAX_SKIP:
            raise ValueError("skip must be in [0, %d] samples (got %d)" % (MAX_SKIP, skip))
        import torch
        ids_dev = isinstance(ids, torch.Tensor) and ids.is_cuda
        if hasattr(at, "event_samples") and hasattr(at, "fired_ids"):
            if not at.timed:
                raise ValueError("at= needs a timed detector (timed=True): an untimed one has no positions")
            if int(at.device) != self.device:
                raise ValueError("the detector is on cuda:%d, the endpointer on cuda:%d" % (at.device, self.device))
            bound = [e for e in (getattr(at, "engine", None), getattr(at, "_arb_engine", None)) if e is not None]
            if any(e is not self.engine for e in bound):
                raise ValueError("the detector serves another engine than this endpointer's")
            if not ids_dev or ids.numel() != at.capacity:
                raise ValueError("with a detector, ids must be a CUDA int32 tensor of its %d slots (passed, confirmed or fired_ids)"
                                 % at.capacity)
            at = at.event_samples
        if isinstance(at, torch.Tensor) and at.is_cuda:
            if not ids_dev:
                raise ValueError("ids and positions must both be host sequences or both CUDA tensors")
            if (ids.dtype != torch.int32 or ids.dim() != 1 or not ids.is_contiguous() or ids.device.index != self.device
                    or at.dtype != torch.int64 or at.dim() != 1 or not at.is_contiguous() or at.device.index != self.device):
                raise ValueError("device ids and positions must be contiguous 1-D CUDA int32 and int64 tensors on cuda:%d" % self.device)
            if at.numel() != ids.numel():
                raise ValueError("ids and positions differ in length (%d, %d)" % (ids.numel(), at.numel()))
            self._check(self._L.mww_endpointer_arm_at_device(self._ep, ids.data_ptr(), at.data_ptr(), ids.numel(), skip, self._stream()))
            return
        if ids_dev or isinstance(at, torch.Tensor):
            raise ValueError("ids and positions must both be host sequences or both CUDA tensors")
        a = _record_ids(ids, "stream ids")
        if a.size and (a.min() < 0 or a.max() >= self.engine.n_streams):
            raise ValueError("stream ids must be in [0, %d)" % self.engine.n_streams)
        p = np.asarray(at)
        if p.ndim != 1 or (p.size and p.dtype.kind not in "iu") or p.size != a.size:
            raise ValueError("positions must be a 1-D integer sequence beside the ids")
        p = np.ascontiguousarray(p, np.int64)
        self._check(self._L.mww_endpointer_arm_at(self._ep, a.ctypes.data, p.ctypes.data, a.size, skip, self._stream()))

    @property
    def positioned(self) -> bool:
        """whether the endpointer runs the positioned kernels: after its first arm(at=...), a loaded mute or an import of
        positioned records"""
        return bool(self.layout().pad)

    def mutes(self) -> np.ndarray:
        """every row's mute word (include/mww.h, "positioned arm"): bits 0 .. 29 the steps still muted, bit 30 set while a
        row armed at a position with nothing replayed has taken no step.  Synchronous."""
        out = np.zeros(self.n_rows, np.int32)
        self._check(self._L.mww_endpointer_get_mutes(self._ep, out.ctypes.data if self.n_rows else None))
        return out

    def disarm(self, ids) -> None:
        """Cancel the listed streams' commands without an event (host ids)"""
        self._ids_call(ids, "mww_endpointer_disarm", None)

    def reset(self, ids=None) -> None:
        """Fresh VAD and segmenter state for all rows (None: also takes the engine's counters as the new baseline, the call to
        make after engine.reset() or reset_frontend()) or the listed GLOBAL stream ids (host, or CUDA int32 such as
        ended_ids): call it with the ids the engine resets."""
        self._ids_call(ids, "mww_endpointer_reset", "mww_endpointer_reset_device", allow_all=True)

    def commands(self, pre: int = 0, post: int = 0, max_samples: int = 160000, out=None, lengths=None):
        """-> (clips, lengths): CUDA int16 [capacity, max_samples] and int32 [capacity].  Row i is event slot i's command,
        samples [start_sample - pre, end) of its stream's history with end = min(speech_end_sample + post, end_sample) for
        END_OF_SPEECH and end_sample otherwise, capped at max_samples; zeros outside the ring and past the length, and
        length 0 in unused slots.  Call it before drain() and before the streams are reset.  Ordered on the current CUDA
        stream, one launch, no host synchronisation."""
        import torch
        pre, post, max_samples = _int(pre, "pre"), _int(post, "post"), _int(max_samples, "max_samples")
        if pre < 0 or post < 0:
            raise ValueError("pre and post must not be negative")
        if not 0 <= max_samples <= MAX_AUDIO_HISTORY:
            raise ValueError("max_samples must be in [0, %d] (got %d)" % (MAX_AUDIO_HISTORY, max_samples))
        dev = torch.device("cuda", self.device)
        if out is None:
            out = torch.empty((self.capacity, max_samples), dtype=torch.int16, device=dev)
        elif (not isinstance(out, torch.Tensor) or out.dtype != torch.int16 or out.device != dev or out.dim() != 2
              or out.shape[0] != self.capacity or out.shape[1] < max_samples or (out.shape[1] > 1 and out.stride(1) != 1)):
            raise ValueError("out must be a CUDA int16 tensor [capacity=%d, >= %d] with contiguous rows on %s" % (self.capacity, max_samples, dev))
        if lengths is None:
            lengths = torch.empty(self.capacity, dtype=torch.int32, device=dev)
        elif (not isinstance(lengths, torch.Tensor) or lengths.dtype != torch.int32 or lengths.device != dev
              or lengths.shape != (self.capacity,) or not lengths.is_contiguous()):
            raise ValueError("lengths must be a contiguous CUDA int32 tensor [capacity=%d] on %s" % (self.capacity, dev))
        stride = out.stride(0) if self.capacity > 1 else max(out.shape[1], max_samples)
        self._check(self._L.mww_endpointer_read_commands(self._ep, self.engine._h, pre, post, max_samples, out.data_ptr(), stride,
                                                         lengths.data_ptr(), self._stream()))
        return out[:, :max_samples], lengths

    def _drain_slots(self):
        buf = np.zeros(self.capacity, ENDPOINT_EVENT_DTYPE)
        n = ctypes.c_longlong(0)
        self._check(self._L.mww_endpointer_drain(self._ep, buf.ctypes.data, self.capacity, ctypes.byref(n), self._stream()))
        return buf[:min(n.value, self.capacity)], n.value

    def drain(self):
        """-> (events, dropped): the commands that ended since the last drain (ENDPOINT_EVENT_DTYPE) sorted by (end_sample,
        stream), and how many more ended than `capacity` could hold.  Waits for the current CUDA stream; clears the event
        buffer and ended_ids."""
        ev, n = self._drain_slots()
        return ev[np.lexsort((ev["stream"], ev["end_sample"]))], max(n - self.capacity, 0)

    def layout(self) -> "_lib.MwwEndpointerLayout":
        """record size, rule window, stride, hop and baseline (mww_get_endpointer_layout; no device work)"""
        out = _lib.MwwEndpointerLayout()
        self._check(self._L.mww_get_endpointer_layout(self._ep, ctypes.byref(out)))
        return out

    def _record_ids(self, stream_ids) -> np.ndarray:
        a = _record_ids(stream_ids, "stream ids")
        if a.size and (a.min() < 0 or a.max() >= self.engine.n_streams):
            raise ValueError("stream ids must be in [0, %d)" % self.engine.n_streams)
        return a

    def export_streams(self, stream_ids) -> EndpointerRecords:
        """The rows of the listed GLOBAL stream ids (host; an id may appear twice) as packed records on this endpointer's
        device, ordered on the current CUDA stream in one launch (mww_export_endpointer_rows).  A stream outside the model's
        stream set exports a zero record.  The endpointer must be up to date with its engine (update() after the engine's
        last call) and does not change; drain() first, since events do not move."""
        import torch
        ids = self._record_ids(stream_ids)
        data = torch.empty((ids.size, int(self.layout().record_bytes)), dtype=torch.uint8, device=torch.device("cuda", self.device))
        layout = _lib.MwwEndpointerLayout()
        self._check(self._L.mww_export_endpointer_rows(self._ep, ids.ctypes.data, ids.size, data.data_ptr() if ids.size else None,
                                                       ctypes.byref(layout), self._stream()))
        return EndpointerRecords(data, layout)

    def import_streams(self, stream_ids, records: EndpointerRecords) -> None:
        """Stream stream_ids[i] (GLOBAL, host, each at most once) takes records.data[i] (mww_import_endpointer_rows): a member
        takes the row, armed under its new id with its positions rebased onto this endpointer's axis (a record of a
        non-member resets it); a non-member ignores the record; unlisted rows keep every byte.  The records' vad_window,
        stride, hop and baseline buffered / pending rows must equal this endpointer's, and it must be up to date with its
        engine.  An arm after the move replays at most min(lookback_steps, steps this endpointer consumed since create or
        its last whole reset): update it for lookback_steps calls before a move for a full-depth replay."""
        import torch
        ids = self._record_ids(stream_ids)
        if np.unique(ids).size != ids.size:
            raise ValueError("a stream id is listed twice")
        data, layout = records.data, records.layout
        if not isinstance(layout, _lib.MwwEndpointerLayout):
            raise ValueError("records.layout must be a MwwEndpointerLayout")
        if (not isinstance(data, torch.Tensor) or data.dtype != torch.uint8 or data.dim() != 2 or data.shape[0] != ids.size
                or data.shape[1] != layout.record_bytes or not data.is_contiguous() or data.device != torch.device("cuda", self.device)):
            raise ValueError("records.data must be a contiguous uint8 tensor [len(ids)=%d, record_bytes=%d] on cuda:%d"
                             % (ids.size, layout.record_bytes, self.device))
        self._check(self._L.mww_import_endpointer_rows(self._ep, ids.ctypes.data, ids.size, data.data_ptr() if ids.size else None,
                                                       ctypes.byref(layout), self._stream()))

    _ROW_FIELDS = (("seen", np.int64), ("flags", np.uint64), ("armed", np.int32), ("elapsed", np.int32), ("run", np.int32),
                   ("silence", np.int32), ("heard", np.int32), ("start_sample", np.int64), ("speech_end_sample", np.int64))

    def state_dict(self) -> dict:
        """every row's state (hist [n_rows, vad_window - 1] oldest first, seen, flags, armed, elapsed, run, silence, heard,
        start_sample, speech_end_sample, mute) and the baseline (samples_seen, buffered, pending), steps and positions [64].
        Synchronous."""
        d = {"hist": np.zeros((self.n_rows, self.vad_window - 1), np.float32)}
        d.update({k: np.zeros(self.n_rows, t) for k, t in self._ROW_FIELDS})
        st = _lib.MwwEndpointState()
        st.hist = d["hist"].ctypes.data if d["hist"].size else None
        for k, _ in self._ROW_FIELDS:
            setattr(st, k, d[k].ctypes.data if self.n_rows else None)
        self._check(self._L.mww_endpointer_get_state(self._ep, ctypes.byref(st)))
        for k in ("samples_seen", "buffered", "pending", "steps"):
            d[k] = int(getattr(st, k))
        d["positions"] = np.ctypeslib.as_array(st.positions).copy()
        d["mute"] = self.mutes()
        return d

    def load_state_dict(self, d: dict) -> None:
        """the inverse of state_dict (synchronous); refusals as mww_endpointer_set_state.  A dict without `mute` loads zero
        mutes.  Nonzero mutes make the endpointer positioned; zero mutes leave a plain endpointer plain."""
        hist = np.ascontiguousarray(d["hist"], np.float32)
        mute = np.ascontiguousarray(d.get("mute", np.zeros(self.n_rows, np.int32)), np.int32)
        if mute.shape != (self.n_rows,) or (mute < 0).any() or ((mute & (MUTE_PLACED - 1)) > MAX_SKIP).any():
            raise ValueError("mute must hold one word per row: a count in [0, 2^22], and bit 30")
        rows = {k: np.ascontiguousarray(d[k], t) for k, t in self._ROW_FIELDS}
        if hist.shape != (self.n_rows, self.vad_window - 1) or any(a.shape != (self.n_rows,) for a in rows.values()):
            raise ValueError("state arrays must have the endpointer's shapes")
        pos = np.ascontiguousarray(d["positions"], np.int64)
        if pos.shape != (64,):
            raise ValueError("positions must hold 64 entries")
        st = _lib.MwwEndpointState()
        st.hist = hist.ctypes.data if hist.size else None
        for k, a in rows.items():
            setattr(st, k, a.ctypes.data if a.size else None)
        for k in ("samples_seen", "buffered", "pending", "steps"):
            setattr(st, k, int(d[k]))
        np.ctypeslib.as_array(st.positions)[:] = pos
        self._check(self._L.mww_endpointer_set_state(self._ep, ctypes.byref(st)))
        if mute.any() or self.positioned:
            self._check(self._L.mww_endpointer_set_mutes(self._ep, mute.ctypes.data if mute.size else None))
