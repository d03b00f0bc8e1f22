"""GPU detection post-processing: the step right after `Model.predict_spectrogram` in the reference's
evaluation harness (microwakeword/test.py).  Same function names / arguments as the reference where it has
a function; the arithmetic runs in libmww_b200.so (csrc/mww_detect.cu) so that only detection counts and
scores -- not every probability -- have to leave the GPU.

    compute_false_accepts_per_hour(tracks, cutoffs, ignore_slices_after_accept=75, stride=1, step_s=0.02)
        == microwakeword.test.compute_false_accepts_per_hour (test.py:94-137) applied to the moving averages
           of `tracks` (pass window=1 to feed already-averaged tracks like the reference call site does)
    moving_average(tracks, window=5)          test.py:337-341
    positive_scores(tracks, window=5, ignore) test.py:364-373
    false_rejection_rates(scores, cutoffs)    test.py:376-381
    generate_roc_curve(faph, frr, cutoffs)    test.py:140-204 (same name, arguments and quirks)
    streaming_model_roc(model, ambient, positives, ...)   the body of test.py:293-403 on spectrogram tracks

Live, the same rule runs per stream with its state carried across calls:

    StreamDetector(n_rows, cutoff, window=5, cooldown_slices=25)   probabilities in (update), detections out (drain)
    MultiModelDetector(engine, cutoffs, windows, cooldown_slices, vad)   the same for every model of a MultiModelEngine in
                                                                       one launch, wake words gated by a VAD model
    set_cutoffs(...)                                                   either one: each stream's own sensitivity
    export_rows / import_rows, export_streams / import_streams         either one: rows moved as packed device records
"""

from __future__ import annotations

import ctypes

import numpy as np

from . import _lib
from .engine import WINDOW


class _Packed:
    """Tracks already on the device: track i is flat[offsets[i] : offsets[i] + lengths[i]] (the layout
    Model._predict_spectrograms_device returns).  Accepted wherever a list of tracks is, so the detection kernels read
    the probabilities in place."""

    def __init__(self, flat, offsets, lengths):
        self.flat = flat
        self.offsets = np.ascontiguousarray(offsets, np.int64)
        self.lengths = np.ascontiguousarray(lengths, np.int32)

    def __len__(self):
        return self.lengths.size


def _pack(tracks, device):
    import torch
    if isinstance(tracks, _Packed):       # the model may live on another GPU than the detection kernels: bring the buffer over
        return (tracks.flat.to(device), torch.from_numpy(tracks.offsets).to(device), torch.from_numpy(tracks.lengths).to(device), tracks.lengths)
    lengths = np.asarray([len(t) for t in tracks], np.int32)
    offsets = np.zeros(len(tracks), np.int64)
    if len(tracks) > 1:
        offsets[1:] = np.cumsum(lengths[:-1], dtype=np.int64)
    if len(tracks) and all(isinstance(t, torch.Tensor) for t in tracks):
        flat = torch.cat([t.to(device=device, dtype=torch.float32).reshape(-1) for t in tracks]) if len(tracks) else torch.zeros(0, device=device)
    else:
        flat = torch.from_numpy(np.concatenate([np.asarray(t, np.float32).reshape(-1) for t in tracks]) if len(tracks) else np.zeros(0, np.float32)).to(device)
    return flat, torch.from_numpy(offsets).to(device), torch.from_numpy(lengths).to(device), lengths


def _stream(device):
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def moving_average(tracks, window: int = 5, device: int = 0):
    """list of 1-D probability tracks -> list of float32 numpy arrays (len - window + 1 each)."""
    import torch
    dev = torch.device("cuda", device)
    flat, offs, lens_d, lens = _pack(tracks, dev)
    out_len = np.maximum(lens.astype(np.int64) - window + 1, 0)
    out_off = np.zeros(len(tracks), np.int64)
    if len(tracks) > 1:
        out_off[1:] = np.cumsum(out_len[:-1])
    out = torch.empty(max(int(out_len.sum()), 1), dtype=torch.float32, device=dev)
    rc = _lib.lib().mww_moving_average(flat.data_ptr(), offs.data_ptr(), lens_d.data_ptr(), len(tracks), int(lens.max()) if len(tracks) else 0, window,
                                       out.data_ptr(), torch.from_numpy(out_off).to(dev).data_ptr(), _stream(dev))
    if rc != 0:
        raise _lib.MwwError(rc, "mww_moving_average failed")
    host = out.cpu().numpy()
    return [host[o:o + n].copy() for o, n in zip(out_off, out_len)]


def false_accept_counts(tracks, cutoffs, ignore_slices_after_accept: int = 75, window: int = 1, device: int = 0) -> np.ndarray:
    """int32 [n_tracks, n_cutoffs] detections (cooldown rule of test.py:120-135) on the `window`-point moving average."""
    import torch
    dev = torch.device("cuda", device)
    flat, offs, lens_d, _ = _pack(tracks, dev)
    cut = torch.from_numpy(np.ascontiguousarray(cutoffs, np.float64)).to(dev)
    counts = torch.zeros((max(len(tracks), 1), cut.numel()), dtype=torch.int32, device=dev)
    rc = _lib.lib().mww_false_accept_counts(flat.data_ptr(), offs.data_ptr(), lens_d.data_ptr(), len(tracks), window, cut.data_ptr(), cut.numel(),
                                            int(ignore_slices_after_accept), counts.data_ptr(), _stream(dev))
    if rc != 0:
        raise _lib.MwwError(rc, "mww_false_accept_counts failed")
    return counts.cpu().numpy()[:len(tracks)]


def compute_false_accepts_per_hour(streaming_probabilities_list, cutoffs, ignore_slices_after_accept: int = 75, stride: int = 1,
                                   step_s: float = 0.02, window: int = 1, device: int = 0) -> np.ndarray:
    """Drop-in for microwakeword.test.compute_false_accepts_per_hour (test.py:94-137).  With the default window=1 the
    tracks are used as given (the reference passes moving averages); window=5 fuses test.py:337-341 into the same pass,
    in which case the duration is counted on the averaged length like the reference does."""
    cutoffs = np.asarray(cutoffs, np.float64)
    counts = false_accept_counts(streaming_probabilities_list, cutoffs, ignore_slices_after_accept, window, device)
    tracks = streaming_probabilities_list
    lengths = tracks.lengths if isinstance(tracks, _Packed) else [len(t) for t in tracks]
    duration_h = 0
    for n in lengths:
        duration_h += max(int(n) - window + 1, 0) * stride * step_s / 3600.0
    return counts.sum(0).astype(np.float64) / duration_h


def positive_scores(tracks, window: int = 5, ignore_slices_after_accept: int = 25, device: int = 0) -> np.ndarray:
    """float32 [n_tracks]: max of the moving average after skipping the first `ignore` probabilities (test.py:364-373)."""
    import torch
    dev = torch.device("cuda", device)
    flat, offs, lens_d, _ = _pack(tracks, dev)
    out = torch.empty(max(len(tracks), 1), dtype=torch.float32, device=dev)
    rc = _lib.lib().mww_positive_scores(flat.data_ptr(), offs.data_ptr(), lens_d.data_ptr(), len(tracks), window, int(ignore_slices_after_accept),
                                        out.data_ptr(), _stream(dev))
    if rc != 0:
        raise _lib.MwwError(rc, "mww_positive_scores failed")
    return out.cpu().numpy()[:len(tracks)]


def accuracy_counts(tracks, min_gap: int, device: int = 0):
    """Per track, the rule of microwakeword.test.tflite_model_accuracy (test.py:452-484): (int32 [n_tracks] count of
    0.5 crossings prev <= 0.5 < p at index j with j - last > min_gap, prev and last restarting at 0 on every track and
    last = j after each counted crossing; bool [n_tracks] last probability > 0.5, False for an empty track)."""
    import torch
    dev = torch.device("cuda", device)
    flat, offs, lens_d, _ = _pack(tracks, dev)
    out = torch.empty((2, max(len(tracks), 1)), dtype=torch.int32, device=dev)
    rc = _lib.lib().mww_accuracy_counts(flat.data_ptr(), offs.data_ptr(), lens_d.data_ptr(), len(tracks), int(min_gap),
                                        out[0].data_ptr(), out[1].data_ptr(), _stream(dev))
    if rc != 0:
        raise _lib.MwwError(rc, "mww_accuracy_counts failed")
    host = out.cpu().numpy()[:, :len(tracks)]
    return host[0].copy(), host[1].astype(bool)


def model_probabilities(model, spectrograms, device: int = 0):
    """The probabilities of `spectrograms` fed one after another to `model`, as the reference's harness feeds them
    (one model, state carried from track to track).  A microwakeword_b200 Model runs them as one batched pass and the
    result stays on the GPU (a packed form every function of this module accepts); an object that has only
    predict_spectrogram is called once per track."""
    spectrograms = list(spectrograms)
    if hasattr(model, "_predict_spectrograms_device"):
        return _Packed(*model._predict_spectrograms_device(spectrograms))
    if hasattr(model, "predict_spectrograms"):
        return [np.asarray(p, np.float32) for p in model.predict_spectrograms(spectrograms)]
    return [np.asarray(model.predict_spectrogram(t), np.float32) for t in spectrograms]


def _split(tracks, k):
    """(tracks[:k], tracks[k:]) for a list or a packed form (views of the same device buffer)."""
    if isinstance(tracks, _Packed):
        return (_Packed(tracks.flat, tracks.offsets[:k], tracks.lengths[:k]), _Packed(tracks.flat, tracks.offsets[k:], tracks.lengths[k:]))
    return tracks[:k], tracks[k:]


def false_rejection_rates(positive_sample_scores, cutoffs) -> np.ndarray:
    """test.py:376-381: 1 - (scores strictly above the cutoff) / (number of positive samples), per cutoff."""
    s = np.asarray(positive_sample_scores, np.float64).reshape(-1)
    if s.size == 0:
        raise ValueError("false_rejection_rates: no positive samples")
    c = np.asarray(cutoffs, np.float64).reshape(-1)
    return 1.0 - (s[None, :] > c[:, None]).sum(1) / float(s.size)


def generate_roc_curve(false_accepts_per_hour, false_rejections, cutoffs, max_faph: float = 2.0):
    """Drop-in for microwakeword.test.generate_roc_curve (test.py:140-204): (faph, false-rejection rate, cutoff) coordinates
    in ascending faph.  Host-side (101 cutoffs).  The reference's quirks are kept on purpose -- callers compare AUC numbers
    across tools: the point at max_faph takes the rejection rate of the last cutoff ABOVE max_faph (the reference reads
    index - 1 for both ordinates, test.py:168-171), interpolates with the literal 2.0 (:173), uses the midpoint cutoff
    (:174-176); equal consecutive faph values keep the first point only (:190-196); a curve that never reaches 0 faph is
    closed with (0, 1) at cutoff 0 (:198-202)."""
    faph = np.asarray(false_accepts_per_hour, np.float64).reshape(-1)
    frr = np.asarray(false_rejections, np.float64).reshape(-1)
    cut = np.asarray(cutoffs, np.float64).reshape(-1)
    if not (faph.size == frr.size == cut.size) or faph.size == 0:
        raise ValueError("generate_roc_curve: faph, false_rejections and cutoffs must have the same non-zero length")
    above = faph > max_faph
    if above[0]:
        if above.all():
            raise IndexError("generate_roc_curve: every cutoff is above max_faph (the reference walks off the array here too)")
        k = int(np.argmin(above))                                    # first cutoff at or below max_faph
        y_prev = frr[k - 1]
        xs, ys, cs = [max_faph], [(y_prev * (faph[k] - 2.0) + y_prev * (2.0 - faph[k - 1])) / (faph[k] - faph[k - 1])], [(cut[k] + cut[k - 1]) / 2.0]
    else:
        k = 0
        xs, ys, cs = [max_faph], [frr[0]], [cut[0]]
    for i in range(k, frr.size):
        if faph[i] != xs[-1]:
            xs.append(faph[i])
            ys.append(frr[i])
            cs.append(cut[i])
    if xs[-1] > 0:
        xs.append(0.0)
        ys.append(1.0)
        cs.append(0.0)
    return np.asarray(xs[::-1]), np.asarray(ys[::-1]), np.asarray(cs[::-1])


def roc_auc(x_coordinates, y_coordinates) -> float:
    """np.trapz(y, x) as test.py:391 computes it (NumPy 2 renamed the function; the arithmetic is spelled out)."""
    x, y = np.asarray(x_coordinates, np.float64), np.asarray(y_coordinates, np.float64)
    return float(np.sum((x[1:] - x[:-1]) * (y[1:] + y[:-1]) / 2.0))


def streaming_model_roc(model, ambient_spectrograms, positive_spectrograms, stride: int = 3, window_step_ms: float = 10.0,
                        sliding_window_length: int = 5, ignore_slices_after_accept: int = 25, cutoffs=None, device: int = 0):
    """The body of microwakeword.test.tflite_streaming_model_roc (test.py:321-403) on lists of spectrogram tracks: ambient
    tracks -> streaming probabilities -> moving average -> false accepts per hour; positive clips -> score -> false
    rejection rate; ROC coordinates and the area under them.  `model` is a microwakeword_b200.inference.Model (or anything
    with predict_spectrograms or predict_spectrogram); the ambient tracks and then the positive clips go through it in
    that order with the state carried over, as in the reference (model_probabilities).  The detection arithmetic runs on
    the GPU, the ROC bookkeeping on the host.  Returns dict(auc, faph, frr, cutoffs, roc=(x, y, cutoff_at_point))."""
    cutoffs = np.arange(0, 1.01, 0.01) if cutoffs is None else np.asarray(cutoffs, np.float64)          # test.py:343
    ambient_spectrograms = list(ambient_spectrograms)
    probs = model_probabilities(model, ambient_spectrograms + list(positive_spectrograms), device)      # test.py:335-336, :367
    ambient, positives = _split(probs, len(ambient_spectrograms))
    faph = compute_false_accepts_per_hour(ambient, cutoffs, ignore_slices_after_accept, stride=stride, step_s=window_step_ms / 1000.0,
                                          window=sliding_window_length, device=device)                 # :337-352 (average fused)
    scores = positive_scores(positives, sliding_window_length, ignore_slices_after_accept, device)      # :368-373
    scores = scores[~np.isnan(scores)]
    frr = false_rejection_rates(scores, cutoffs)
    x, y, c = generate_roc_curve(faph, frr, cutoffs)
    return dict(auc=roc_auc(x, y), faph=faph, frr=frr, cutoffs=cutoffs, roc=(x, y, c))


# ---- the streaming detector ----------------------------------------------------------------------------------------------
EVENT_DTYPE = np.dtype([("stream", np.int32), ("reserved", np.int32), ("step", np.int64), ("score", np.float32), ("pad", np.int32)])


class _DetectorHandle:
    """owner of one mww_detector_t: destroyed when the detector and every tensor over its buffers are gone"""

    def __init__(self, L, ptr):
        self.L, self.ptr = L, ptr

    def close(self):
        if self.ptr:
            self.L.mww_detector_destroy(self.ptr)
            self.ptr = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class _DeviceArray:
    """a span of a detector's device memory, as torch.as_tensor takes it; the tensor keeps this object, and through it the
    detector's handle, alive"""

    def __init__(self, handle: _DetectorHandle, ptr: int, n: int, typestr: str):
        self.handle = handle
        self.__cuda_array_interface__ = dict(shape=(n,), typestr=typestr, data=(ptr, False), version=2, strides=None)


def _record_ids(ids, what: str) -> np.ndarray:
    """a list, NumPy array or CPU tensor of ids -> contiguous int32 array, or ValueError"""
    if hasattr(ids, "is_cuda"):
        if ids.is_cuda:
            raise ValueError("%s must be in host memory" % what)
        ids = ids.numpy()
    a = np.asarray(ids)
    if a.ndim != 1 or (a.size and (a.dtype == bool or not np.issubdtype(a.dtype, np.integer))):
        raise ValueError("%s must be a 1-D sequence of integers" % what)
    if a.size and (a.min() < np.iinfo(np.int32).min or a.max() > np.iinfo(np.int32).max):
        raise ValueError("%s must fit in int32" % what)
    return np.ascontiguousarray(a, np.int32)


class DetectorRecords:
    """Detector rows exported from a StreamDetector (export_rows) or a MultiModelDetector (export_streams): `data`,
    torch.uint8 [n, record_bytes] on the detector's device, one packed record per listed id (include/mww.h), and `layout`,
    the _lib.MwwDetectorLayout an importing detector must share.  `cutoffs` is each exported id's cutoff: float64 [n] for a
    plain detector, a list of one float64 [n] per model for a models detector (NaN where the stream is not a member and
    for an OFF model).  The records carry no events and no stream map."""

    _SCALARS = ("record_bytes", "multi", "n_models")
    _ARRAYS = ("role", "window", "cooldown_slices")

    def __init__(self, data, layout, cutoffs):
        self.data, self.layout, self.cutoffs = data, layout, cutoffs

    def save(self, path) -> None:
        """np.savez of the records, the layout's fields and the cutoffs: a checkpoint of some streams' detector rows"""
        fields = {k: np.asarray(getattr(self.layout, k)) for k in self._SCALARS}
        fields.update({k: np.ctypeslib.as_array(getattr(self.layout, k)).copy() for k in self._ARRAYS})
        cut = np.stack(self.cutoffs) if self.layout.multi else np.asarray(self.cutoffs)
        np.savez(path, data=self.data.cpu().numpy(), cutoffs=cut.astype(np.float64), **fields)

    @classmethod
    def load(cls, path, device) -> "DetectorRecords":
        import torch
        layout = _lib.MwwDetectorLayout()
        with np.load(path) as z:
            for k in cls._SCALARS:
                setattr(layout, k, int(z[k]))
            for k in cls._ARRAYS:
                np.ctypeslib.as_array(getattr(layout, k))[:] = z[k]
            data = torch.from_numpy(z["data"]).to(device)
            cut = np.asarray(z["cutoffs"], np.float64)
        return cls(data, layout, [c.copy() for c in cut] if layout.multi else cut.copy())


def timed_dtype(dtype) -> np.dtype:
    """the drain dtype of a timed detector: `dtype` and the int64 `sample`, each event's position on the audio history's axis"""
    return np.dtype(dtype.descr + [("sample", np.int64)])


def grouped_dtype(dtype) -> np.dtype:
    """the drain dtype of a grouped detector: timed_dtype(dtype) and the int32 `group` and `candidates` of each event (group -1
    and candidates 1 for an event of an ungrouped row)"""
    return np.dtype(timed_dtype(dtype).descr + [("group", np.int32), ("candidates", np.int32)])


def arbitrated_dtype(dtype) -> np.dtype:
    """the drain dtype of an arbitrated detector: grouped_dtype(dtype) and the float32 `level` of each event (NaN for an event
    of an ungrouped row); 10 log10(level) is the level in dB"""
    return np.dtype(grouped_dtype(dtype).descr + [("level", np.float32)])


# mww_group_window of include/mww.h: one group slot's window
GROUP_WINDOW_DTYPE = np.dtype([("deadline", np.int64), ("sample", np.int64), ("step", np.int64), ("stream", np.int32), ("score", np.float32),
                               ("candidates", np.int32), ("open", np.int32)])


def _group_list(ids, groups, name):
    """(int32 ids, int32 groups) of one set-groups call, or ValueError: ids a 1-D integer sequence, groups one integer or one per id"""
    i = _record_ids(ids, name)
    g = np.asarray(groups)
    if g.dtype == bool or not (np.issubdtype(g.dtype, np.integer) or g.size == 0):
        raise ValueError("groups must be integers")
    if g.ndim == 0:
        g = np.full(i.size, g, np.int64)
    if g.shape != i.shape:
        raise ValueError("groups must be one value or one per entry of %s (%d)" % (name, i.size))
    if g.size and (g.min() < np.iinfo(np.int32).min or g.max() > np.iinfo(np.int32).max):
        raise ValueError("groups must fit in int32")
    return i, np.ascontiguousarray(g, np.int32)


def _history_clock(engine, model):
    """(samples_seen S, b, hop) of an engine with an audio history, read now: its newest feature row's window ends at history
    sample S - b (include/mww.h, "event positions"); ValueError without a history, on which positions mean nothing"""
    cap, S = engine._audio_history()
    if cap == 0:
        raise ValueError("a timed detector places events on the engine's audio history axis: the engine keeps no audio history "
                         "(set_audio_history)")
    hop = int(engine.hop)
    return S, engine.frontend_buffered - (WINDOW - hop), hop


class _Detector:
    """what both detectors share: ownership of one mww_detector_t, its device views, drain, the reset dispatch and the
    record calls"""

    def _own(self, rc: int, d, device: int, capacity: int) -> None:
        """take the detector a create call returned (rc, d) and make the views of its event buffers"""
        self._check(rc)
        self._handle = _DetectorHandle(self._L, d)
        self.device, self.capacity = int(device), int(capacity)
        count, fired = ctypes.c_void_p(), ctypes.c_void_p()
        self._check(self._L.mww_detector_buffers(self._d, ctypes.byref(count), None, ctypes.byref(fired), None))
        import torch
        dev = torch.device("cuda", self.device)
        with torch.cuda.device(dev):
            # device views: the stream of every event since the last drain (-1 in unused slots), and how many fired
            self.fired_ids = torch.as_tensor(_DeviceArray(self._handle, fired.value, self.capacity, "<i4"), device=dev)
            self.event_count = torch.as_tensor(_DeviceArray(self._handle, count.value, 1, "<i8"), device=dev)
        self.timed = False
        self.event_samples = None
        self.n_groups, self.group_window = 0, 0
        self.arbitrated, self._arb_engine = False, None

    def _time(self) -> None:
        """make the detector timed (mww_time_detector_events) and make event_samples, the device view of the positions"""
        self._check(self._L.mww_time_detector_events(self._d))
        ptr = ctypes.c_void_p()
        self._check(self._L.mww_get_detector_positions(self._d, ctypes.byref(ptr)))
        import torch
        dev = torch.device("cuda", self.device)
        with torch.cuda.device(dev):
            # the position of every event since the last drain on the audio history's axis, slot by slot as fired_ids (-1 in
            # unused slots)
            self.event_samples = torch.as_tensor(_DeviceArray(self._handle, ptr.value, self.capacity, "<i8"), device=dev)
        self.timed = True

    @staticmethod
    def _group_args(timed: bool, groups, group_window) -> None:
        """ValueError unless groups is None, or an integer with timed and an integer group_window"""
        if groups is None:
            return
        if not timed:
            raise ValueError("groups need a timed detector (timed=True): the rule places every detection on the audio history's axis")
        for v, name in ((groups, "groups"), (group_window, "group_window")):
            if isinstance(v, bool) or not isinstance(v, (int, np.integer)):
                raise ValueError("%s must be an integer (got %r)" % (name, v))

    def _group(self, groups, group_window) -> None:
        """make a timed detector grouped (mww_group_detector_events): `groups` groups, windows of `group_window` samples"""
        if groups is None:
            return
        self._check(self._L.mww_group_detector_events(self._d, int(groups), int(group_window)))
        self.n_groups, self.group_window = int(groups), int(group_window)

    @property
    def grouped(self) -> bool:
        return self.n_groups > 0

    def _n_group_slots(self) -> int:
        return self.n_groups * (sum(r == _lib.MWW_DETECT_WAKE for r in self.roles) if hasattr(self, "roles") else 1)

    def _arbitrate(self, engine, speech_samples, noise_samples) -> None:
        """bind a grouped detector's arbitration to `engine`'s audio history (mww_arbitrate_detector_groups)"""
        for v, name in ((speech_samples, "speech_samples"), (noise_samples, "noise_samples")):
            if isinstance(v, bool) or not isinstance(v, (int, np.integer)):
                raise ValueError("%s must be an integer (got %r)" % (name, v))
        if not self.grouped:
            raise ValueError("arbitration picks the winner of a group: make the detector with groups=n first")
        self._check(self._L.mww_arbitrate_detector_groups(self._d, engine._h, int(speech_samples), int(noise_samples)))
        self.arbitrated, self._arb_engine = True, engine
        self.speech_samples, self.noise_samples = int(speech_samples), int(noise_samples)

    def group_levels(self) -> np.ndarray:
        """float32 [group slots]: the level of each open window's best candidate (slots as group_windows'); waits for the
        device"""
        out = np.zeros(self._n_group_slots(), np.float32)
        self._check(self._L.mww_get_detector_group_levels(self._d, out.ctypes.data))
        return out

    def flush(self) -> None:
        """Emit every open group window now (mww_flush_detector_groups): before a final drain, or before moving streams out
        of this detector.  Ordered on the current CUDA stream; one launch."""
        self._check(self._L.mww_flush_detector_groups(self._d, self._cuda_stream()))

    def group_windows(self) -> np.ndarray:
        """GROUP_WINDOW_DTYPE [group slots]: each group's open window (slot g n_wake + w of a models detector, w the WAKE model's
        index among the WAKE models); waits for the device"""
        out = np.zeros(self._n_group_slots(), GROUP_WINDOW_DTYPE)
        self._check(self._L.mww_get_detector_group_windows(self._d, out.ctypes.data))
        return out

    def _group_state(self, d: dict) -> dict:
        if self.grouped:
            d["groups"] = self.groups
            d["group_windows"] = self.group_windows()
        if self.arbitrated:
            d["group_levels"] = self.group_levels()
        return d

    def _load_group_state(self, d: dict):
        """the checked (groups, windows) of a state dict, to apply with _apply_group_state once every other part is checked"""
        if not self.grouped:
            if "groups" in d:
                raise ValueError("the state holds groups; this detector is not grouped")
            return None
        if "groups" not in d or "group_windows" not in d:
            raise ValueError("a grouped detector's state holds groups and group_windows")
        g = np.ascontiguousarray(d["groups"], np.int32)
        w = np.ascontiguousarray(d["group_windows"], GROUP_WINDOW_DTYPE)
        if g.shape != self.groups.shape or w.shape != (self._n_group_slots(),):
            raise ValueError("groups must be [%d] and group_windows [%d]" % (self.groups.size, self._n_group_slots()))
        if g.size and (g.min() < -1 or g.max() >= self.n_groups):
            raise ValueError("groups must be in [-1, %d)" % self.n_groups)
        if not np.isin(w["open"], (0, 1)).all() or (w["candidates"][w["open"] == 1] < 1).any():
            raise ValueError("group_windows: open must be 0 or 1, and an open window needs candidates >= 1")
        if not self.arbitrated:
            if "group_levels" in d:
                raise ValueError("the state holds group_levels; this detector is not arbitrated")
            return g, w, None
        if "group_levels" not in d:
            raise ValueError("an arbitrated detector's state holds group_levels")
        lv = np.ascontiguousarray(d["group_levels"], np.float32)
        if lv.shape != (self._n_group_slots(),):
            raise ValueError("group_levels must be [%d]" % self._n_group_slots())
        if not (np.isfinite(lv).all() and (lv >= 0).all()):
            raise ValueError("group_levels must be finite and not negative")
        return g, w, lv

    def _apply_group_state(self, gw) -> None:
        if gw is None:
            return
        g, w, lv = gw
        ids = np.arange(g.size, dtype=np.int32)
        fn = self._L.mww_set_multi_detector_groups if hasattr(self, "roles") else self._L.mww_set_detector_groups
        self._check(fn(self._d, ids.ctypes.data, g.ctypes.data, g.size, self._cuda_stream()))
        self._check(self._L.mww_set_detector_group_windows(self._d, w.ctypes.data))
        if lv is not None:
            self._check(self._L.mww_set_detector_group_levels(self._d, lv.ctypes.data))

    def _check(self, rc: int) -> None:
        if rc != 0:
            msg = self._L.mww_last_error(None)
            raise _lib.MwwError(rc, msg.decode() if msg else "detector call failed")

    @property
    def _d(self):
        return self._handle.ptr

    def _cuda_stream(self):
        import torch
        return _stream(torch.device("cuda", self.device))

    def close(self):
        """free the detector now; fired_ids and event_count must not be used afterwards"""
        self._handle.close()

    def _drain_slots(self, dtype):
        """(events since the last drain as `dtype` in slot order, events that fired); a timed detector's events carry `sample`
        too (timed_dtype)"""
        buf = np.empty(self.capacity, dtype)
        n = ctypes.c_longlong(0)
        if not self.timed:
            self._check(self._L.mww_detector_drain(self._d, buf.ctypes.data, self.capacity, ctypes.byref(n), self._cuda_stream()))
            return buf[:min(n.value, self.capacity)], n.value
        pos = np.empty(self.capacity, np.int64)
        if self.arbitrated:
            grp, cand, lev = np.empty(self.capacity, np.int32), np.empty(self.capacity, np.int32), np.empty(self.capacity, np.float32)
            self._check(self._L.mww_drain_detector_arbitrated(self._d, buf.ctypes.data, pos.ctypes.data, grp.ctypes.data, cand.ctypes.data,
                                                              lev.ctypes.data, self.capacity, ctypes.byref(n), self._cuda_stream()))
        elif self.grouped:
            grp, cand = np.empty(self.capacity, np.int32), np.empty(self.capacity, np.int32)
            self._check(self._L.mww_drain_detector_groups(self._d, buf.ctypes.data, pos.ctypes.data, grp.ctypes.data, cand.ctypes.data,
                                                          self.capacity, ctypes.byref(n), self._cuda_stream()))
        else:
            self._check(self._L.mww_drain_detector_at(self._d, buf.ctypes.data, pos.ctypes.data, self.capacity, ctypes.byref(n),
                                                      self._cuda_stream()))
        m = min(n.value, self.capacity)
        out = np.empty(m, arbitrated_dtype(dtype) if self.arbitrated else grouped_dtype(dtype) if self.grouped else timed_dtype(dtype))
        for name in dtype.names:
            out[name] = buf[name][:m]
        out["sample"] = pos[:m]
        if self.grouped:
            out["group"], out["candidates"] = grp[:m], cand[:m]
        if self.arbitrated:
            out["level"] = lev[:m]
        return out, n.value

    def _drain(self, dtype, keys):
        """(events since the last drain as `dtype`, sorted by `keys`, most significant first; events dropped)"""
        ev, n = self._drain_slots(dtype)
        return ev[np.lexsort(tuple(ev[k] for k in reversed(keys)))], max(n - self.capacity, 0)

    def layout(self) -> "_lib.MwwDetectorLayout":
        """record size, kind and each model's role, window and cooldown (mww_get_detector_layout; no device work)"""
        out = _lib.MwwDetectorLayout()
        self._check(self._L.mww_get_detector_layout(self._d, ctypes.byref(out)))
        return out

    def _export(self, ids, what: str):
        """(records [n, record_bytes] of the listed ids, their layout), ordered on the current CUDA stream"""
        import torch
        ids = _record_ids(ids, what)
        data = torch.empty((ids.size, int(self.layout().record_bytes)), dtype=torch.uint8, device=torch.device("cuda", self.device))
        layout = _lib.MwwDetectorLayout()
        self._check(self._L.mww_export_detector_rows(self._d, ids.ctypes.data, ids.size, data.data_ptr(), ctypes.byref(layout),
                                                     self._cuda_stream()))
        return ids, data, layout

    def _import(self, ids, records: "DetectorRecords", what: str) -> np.ndarray:
        """the listed ids take the records' state (the cutoffs are the caller's part); -> the ids as int32"""
        import torch
        ids = _record_ids(ids, what)
        data = records.data
        if (not isinstance(data, torch.Tensor) or data.dtype != torch.uint8 or data.dim() != 2 or data.shape[0] != ids.size
                or data.shape[1] != records.layout.record_bytes or not data.is_contiguous() or not data.is_cuda
                or data.device.index != self.device):
            raise ValueError("records.data must be a contiguous uint8 tensor [len(%s)=%d, record_bytes=%d] on cuda:%d"
                             % (what, ids.size, records.layout.record_bytes, self.device))
        self._check(self._L.mww_import_detector_rows(self._d, ids.ctypes.data, ids.size, data.data_ptr(), ctypes.byref(records.layout),
                                                     self._cuda_stream()))
        return ids

    def _reset(self, ids, what: str) -> None:
        """reset all rows (None), or the ids of a contiguous 1-D CUDA int32 tensor or of a host sequence"""
        import torch
        st = self._cuda_stream()
        if ids is None:
            self._check(self._L.mww_detector_reset(self._d, None, 0, st))
        elif isinstance(ids, torch.Tensor) and ids.is_cuda:
            if ids.dtype != torch.int32 or ids.dim() != 1 or not ids.is_contiguous():
                raise ValueError("device %s must be a contiguous 1-D CUDA int32 tensor" % what)
            self._check(self._L.mww_detector_reset_device(self._d, ids.data_ptr(), ids.numel(), st))
        else:
            r = np.ascontiguousarray(ids, np.int32).reshape(-1)
            self._check(self._L.mww_detector_reset(self._d, r.ctypes.data, r.size, st))


class StreamDetector(_Detector):
    """The detection rule of the reference's evaluation (moving average of `window` probabilities above `cutoff`, then
    `cooldown_slices` steps of silence; test.py:337-341, :118-135) for `n_rows` live streams, state carried across calls
    (mww_detector_* of include/mww.h).  A row's events over any sequence of update calls are those of false_accept_counts on
    everything it was given; an event's `step` counts the row's probabilities since its last reset, `score` is the average
    that fired.  It consumes what step() / predict_clip() return and knows nothing else of the engine:

        det = StreamDetector(eng.n_streams, cutoff=0.9)
        det.update(eng.step(chunk))            # nothing leaves the GPU
        events, dropped = det.drain()          # now and then: a few events
        eng.reset(det.fired_ids)               # before a drain: restart the streams that fired, no host round trip

    `stream_ids`: event.stream of each row when it is not the row index (model k of an engine with stream sets scores its
    members in list order: pass MultiModelEngine.streams[k]).  `capacity`: events kept between drains; more are
    counted and dropped.

    `timed=True` places every event on the engine's audio history axis (include/mww.h, "event positions"): update takes the
    engine whose call made the probabilities, drain adds an int64 `sample` field, and event_samples is a device view beside
    fired_ids.  Update right after each engine call, before the next changes its counters, and drain before
    engine.set_audio_history, which restarts the axis:

        eng.set_audio_history(48000)
        det = StreamDetector(eng.n_streams, cutoff=0.9, timed=True)
        det.update(eng.step(chunk), eng)
        clips = eng.audio_history(det.fired_ids, 24000, end=det.event_samples)   # the 1.5 s before each detection

    `groups=n` (timed only) answers a wake word once per household (include/mww.h, "grouped detection"): set_groups puts rows
    in groups [0, n) (-1: none, the default), and of the detections of one group that start within `group_window` samples
    only the best is stored, up to group_window + one step after it fired; drain adds `group` and `candidates`, and flush()
    stores the windows still open.  Every row's state, cooldown included, is what the ungrouped detector's would be.

    arbitrate(engine) makes the household's answer come from the satellite that heard the wake word loudest over its own
    background (include/mww.h, "group arbitration"): each candidate's level is measured from the engine's audio history and
    compared before the score, and drain adds a float32 `level` (NaN for rows of group -1)."""

    def __init__(self, n_rows: int, cutoff: float, window: int = 5, cooldown_slices: int = 25, capacity: int = 65536,
                 stream_ids=None, device: int = 0, timed: bool = False, groups=None, group_window: int = 0):
        self._group_args(timed, groups, group_window)
        self._L = _lib.lib()
        d = ctypes.c_void_p()
        ids = None
        if stream_ids is not None:
            ids = np.ascontiguousarray(stream_ids, np.int32).reshape(-1)
            if ids.size != int(n_rows):
                raise ValueError("stream_ids must name one stream per row")
        rc = self._L.mww_detector_create(int(device), int(n_rows), int(window), float(cutoff), int(cooldown_slices), int(capacity),
                                         ids.ctypes.data if ids is not None else None, ctypes.byref(d))
        self._own(rc, d, device, capacity)
        self.n_rows, self.window, self.cutoff, self.cooldown_slices = int(n_rows), int(window), float(cutoff), int(cooldown_slices)
        if timed:
            self._time()
        self._group(groups, group_window)

    def update(self, probs, engine=None, model=None) -> None:
        """CUDA float32 [n_rows, steps], any row pitch (a slice of a wider buffer is read in place); zero columns: nothing
        happens.  Asynchronous on the current CUDA stream.  A timed detector takes the engine whose call just returned
        `probs` (with `model` = k for probs[k] of a MultiModelEngine) and reads the clock of its steps from the engine's
        counters now; an untimed detector takes neither."""
        import torch
        if not self.timed:
            if engine is not None or model is not None:
                raise ValueError("only a timed detector (timed=True) takes the engine and model")
        else:
            if engine is None:
                raise ValueError("a timed detector needs the engine whose call made the probabilities")
            multi = hasattr(engine, "n_models")
            if multi and (isinstance(model, bool) or not isinstance(model, (int, np.integer)) or not 0 <= model < engine.n_models):
                raise ValueError("model must be a model index in [0, %d) for a MultiModelEngine (got %r)" % (engine.n_models, model))
            if not multi and model is not None:
                raise ValueError("model selects a model of a MultiModelEngine; a StreamEngine has one")
            if self.arbitrated and engine is not self._arb_engine:
                raise ValueError("an arbitrated detector measures the engine it was bound to (arbitrate): update it with that engine")
            S, b, hop = _history_clock(engine, model)
            stride = engine.stride[int(model)] if multi else engine.stride
            g = engine.pending_rows[int(model)] if multi else engine.pending_rows
        if (not isinstance(probs, torch.Tensor) or not probs.is_cuda or probs.dtype != torch.float32 or probs.dim() != 2
                or probs.shape[0] != self.n_rows or probs.device.index != self.device):
            raise ValueError("probs must be a CUDA float32 tensor [n_rows=%d, steps] on device %d" % (self.n_rows, self.device))
        n = probs.shape[1]
        if n == 0:
            return
        if (n > 1 and probs.stride(1) != 1) or (self.n_rows > 1 and probs.stride(0) < n):
            probs = probs.contiguous()
        pitch = probs.stride(0) if self.n_rows > 1 else n
        if self.timed:
            self._check(self._L.mww_update_detector_at(self._d, probs.data_ptr(), n, pitch, S - b - hop * g, hop * stride, _stream(probs.device)))
        else:
            self._check(self._L.mww_detector_update(self._d, probs.data_ptr(), n, pitch, _stream(probs.device)))

    def drain(self):
        """-> (events, dropped): the events since the last drain as a structured array (EVENT_DTYPE, `sample` for a timed
        detector, `group` and `candidates` for a grouped one) sorted by (step, stream), and how many more fired than `capacity` could hold.  Waits for the current CUDA
        stream; clears the event buffer and fired_ids."""
        return self._drain(EVENT_DTYPE, ("step", "stream"))

    def reset(self, rows=None) -> None:
        """Fresh detector state (warm-up and cooldown start again) for all rows (None) or the given ROW indices: a host
        sequence, or a contiguous 1-D CUDA int32 tensor.  Indices out of range are ignored."""
        self._reset(rows, "row indices")

    def state_dict(self) -> dict:
        """{hist [n_rows, window - 1], seen [n_rows], cooldown [n_rows]}, and a grouped detector's groups [n_rows] and
        group_windows (GROUP_WINDOW_DTYPE [groups]), and an arbitrated one's group_levels (float32 [groups])"""
        d = dict(hist=np.zeros((self.n_rows, self.window - 1), np.float32), seen=np.zeros(self.n_rows, np.int64),
                 cooldown=np.zeros(self.n_rows, np.int32))
        self._check(self._L.mww_detector_get_state(self._d, d["hist"].ctypes.data, d["seen"].ctypes.data, d["cooldown"].ctypes.data))
        return self._group_state(d)

    def load_state_dict(self, d: dict) -> None:
        hist = np.ascontiguousarray(d["hist"], np.float32)
        seen = np.ascontiguousarray(d["seen"], np.int64)
        cooldown = np.ascontiguousarray(d["cooldown"], np.int32)
        if hist.shape != (self.n_rows, self.window - 1) or seen.shape != (self.n_rows,) or cooldown.shape != (self.n_rows,):
            raise ValueError("state must be hist [n_rows, window - 1], seen [n_rows], cooldown [n_rows]")
        gw = self._load_group_state(d)
        self._check(self._L.mww_detector_set_state(self._d, hist.ctypes.data, seen.ctypes.data, cooldown.ctypes.data))
        self._apply_group_state(gw)

    def arbitrate(self, engine, speech_samples: int = 12000, noise_samples: int = 8000) -> None:
        """Pick each group window's winner by level, then score (mww_arbitrate_detector_groups), for good: a candidate at
        position P is measured over the speech span [P - speech_samples, P) and the noise span of noise_samples before it, both
        read from `engine`'s audio history (the engine every update takes; the rows' streams are its streams), and its level
        is (mean-removed power of speech + 1) / (that of noise + 1).  10 log10(level) is the level in dB.  The defaults, 0.75 s
        of speech after 0.5 s of noise, are guesses: nobody has measured which spans pick the nearest device best in real
        rooms.  Only on a grouped detector that holds no events (after create, or a drain before any update)."""
        self._arbitrate(engine, speech_samples, noise_samples)

    def set_groups(self, rows, groups) -> None:
        """Put the listed ROW indices in `groups` (one value or one per row; -1: no group) (mww_set_detector_groups).  Ordered
        on the current CUDA stream: updates after it use the new groups.  An open window keeps its candidates."""
        r, g = _group_list(rows, groups, "rows")
        self._check(self._L.mww_set_detector_groups(self._d, r.ctypes.data, g.ctypes.data, r.size, self._cuda_stream()))

    @property
    def groups(self) -> np.ndarray:
        """int32 [n_rows]: every row's group, -1 for none"""
        out = np.empty(self.n_rows, np.int32)
        self._check(self._L.mww_get_detector_groups(self._d, out.ctypes.data))
        return out


    def set_cutoffs(self, rows, cutoffs) -> None:
        """Give the listed ROW indices their own cutoffs (mww_set_detector_cutoffs): `cutoffs` is one value or one per row.
        The first call switches the detector to per-row mode, every other row keeping the create-time cutoff.  Ordered on
        the current CUDA stream: updates made before it use the old cutoffs, updates after it the new ones.  The state and
        resets are unaffected."""
        r, c = _cutoff_list(rows, cutoffs, "rows")
        self._check(self._L.mww_set_detector_cutoffs(self._d, r.ctypes.data, c.ctypes.data, r.size, self._cuda_stream()))

    @property
    def cutoffs(self) -> np.ndarray:
        """float64 [n_rows]: every row's cutoff (the create-time one everywhere until set_cutoffs is called)"""
        out = np.empty(self.n_rows, np.float64)
        self._check(self._L.mww_get_detector_cutoffs(self._d, out.ctypes.data))
        return out

    def export_rows(self, rows) -> DetectorRecords:
        """The state of the listed ROW indices (hist, seen, cooldown) as packed records on this detector's device, ordered on
        the current CUDA stream in one launch (mww_export_detector_rows), with each row's cutoff beside them.  A row may be
        listed twice.  The detector does not change; events stay where they are (drain before moving)."""
        ids, data, layout = self._export(rows, "rows")
        return DetectorRecords(data, layout, self.cutoffs[ids])

    def import_rows(self, rows, records: DetectorRecords) -> None:
        """Row rows[i] takes the state of records.data[i] (mww_import_detector_rows) and continues bit for bit as the exported
        row would have, its events reporting this detector's stream map.  Every other row is untouched.  Rows whose
        exported cutoff differs from theirs get it (one set_cutoffs call, on the same CUDA stream), so two uniform detectors
        with the same cutoff stay uniform.  Records of another kind, window or cooldown, out-of-range or duplicate rows:
        MwwError with nothing changed; a malformed row list or records on another device: ValueError."""
        if records.layout.multi == 0:
            c = np.asarray(records.cutoffs, np.float64)
            if c.shape != (records.data.shape[0],):
                raise ValueError("records.cutoffs must hold one cutoff per record")
        ids = self._import(rows, records, "rows")
        c = np.asarray(records.cutoffs, np.float64)
        diff = np.flatnonzero(c != self.cutoffs[ids])
        if diff.size:
            self.set_cutoffs(ids[diff], c[diff])


def _cutoff_list(ids, cutoffs, name):
    """(int32 ids, float64 cutoffs) of one set-cutoffs call, or ValueError: ids a 1-D integer sequence, cutoffs one finite
    real value or one per id"""
    i = np.asarray(ids)
    if i.ndim != 1 or not (np.issubdtype(i.dtype, np.integer) or i.size == 0):
        raise ValueError("%s must be a 1-D sequence of integers" % name)
    if i.size and (i.min() < np.iinfo(np.int32).min or i.max() > np.iinfo(np.int32).max):
        raise ValueError("%s must fit in int32" % name)
    c = np.asarray(cutoffs)
    if c.dtype == bool or not (np.issubdtype(c.dtype, np.floating) or np.issubdtype(c.dtype, np.integer)):
        raise ValueError("cutoffs must be real numbers")
    if c.ndim == 0:
        c = np.full(i.size, c, np.float64)
    if c.shape != i.shape:
        raise ValueError("cutoffs must be one value or one per entry of %s (%d)" % (name, i.size))
    c = np.ascontiguousarray(c, np.float64)
    if not np.isfinite(c).all():
        raise ValueError("cutoffs must be finite")
    return np.ascontiguousarray(i, np.int32), c


# ---- the multi-model streaming detector ----------------------------------------------------------------------------------
MODEL_EVENT_DTYPE = np.dtype([("stream", np.int32), ("model", np.int32), ("step", np.int64), ("score", np.float32), ("pad", np.int32)])


def _per_model(value, K, name):
    v = list(value) if isinstance(value, (list, tuple, np.ndarray)) else [value] * K
    if len(v) != K:
        raise ValueError("%s must be one value or one per model (%d)" % (name, K))
    return v


class MultiModelDetector(_Detector):
    """One detector over the K models of a MultiModelEngine (mww_multi_detector_create of include/mww.h): each model WAKE
    (the StreamDetector rule), the VAD or OFF, every model's probabilities of a call in one launch, one event stream.  A WAKE
    model fires only on streams whose VAD row is active (the VAD's moving average above its cutoff); without a VAD each
    WAKE model is exactly a StreamDetector over its stream set.

        det = MultiModelDetector(eng, cutoffs=[0.97, 0.95, 0.5], windows=[5, 5, 10], vad=2)
        det.update(eng.step(chunk))            # one launch for every model
        events, dropped = det.drain()          # now and then: events with a `model` field
        eng.reset(det.fired_ids)               # the streams on which any wake word fired, global ids
        det.reset(det.fired_ids)

    `cutoffs[k] = None` makes model k OFF; `windows` and `cooldown_slices` are one value or one per model (the VAD's
    cooldown is not used).  The detector copies the engine's strides and stream sets at creation and reads its pending rows
    then and after every update: it must see every call the engine makes, and after `engine.reset()` it needs `reset()`;
    after `engine.set_streams` make a new one and import every stream from the old one, so that the streams that stay
    keep their rows and cutoffs:

        new = MultiModelDetector(eng, ...)     # the same rules
        all_ids = np.arange(eng.n_streams)
        new.import_streams(all_ids, det.export_streams(all_ids))

    `timed=True` places every event on the engine's audio history axis, as StreamDetector's does: update reads the clock from
    the engine, which must keep an audio history, drain adds `sample` and event_samples is the device view.

    `groups=n` (timed only) groups streams as StreamDetector's does, per (group, WAKE model): set_groups takes global stream
    ids, one group per stream for all its wake words.  arbitrate(engine) picks each window's winner by level, as
    StreamDetector.arbitrate does."""

    def __init__(self, engine, cutoffs, windows=5, cooldown_slices: int = 25, vad=None, capacity: int = 65536, timed: bool = False,
                 groups=None, group_window: int = 0):
        self._group_args(timed, groups, group_window)
        K = engine.n_models
        cutoffs = _per_model(cutoffs, K, "cutoffs")
        windows = _per_model(windows, K, "windows")
        cooldowns = _per_model(cooldown_slices, K, "cooldown_slices")
        if vad is not None and not 0 <= int(vad) < K:
            raise ValueError("vad must be a model index in [0, %d)" % K)
        if vad is not None and cutoffs[int(vad)] is None:
            raise ValueError("the VAD model needs a cutoff")
        rules = (_lib.MwwDetectRule * K)()
        for k in range(K):
            role = (_lib.MWW_DETECT_OFF if cutoffs[k] is None else
                    _lib.MWW_DETECT_VAD if vad is not None and k == int(vad) else _lib.MWW_DETECT_WAKE)
            rules[k] = _lib.MwwDetectRule(role, int(windows[k]), int(cooldowns[k]), 0, 0.0 if cutoffs[k] is None else float(cutoffs[k]))
        self._L = _lib.lib()
        d = ctypes.c_void_p()
        self._own(self._L.mww_multi_detector_create(engine._h, rules, int(capacity), ctypes.byref(d)), d, engine.device, capacity)
        self.engine, self.n_models = engine, K
        self.roles = [r.role for r in rules]
        self.vad = None if vad is None else int(vad)
        self.windows = [int(w) for w in windows]
        self.cutoffs = [None if c is None else float(c) for c in cutoffs]
        self.cooldown_slices = [int(c) for c in cooldowns]
        self.streams = [s.copy() for s in engine.streams]
        self._pending = list(engine.pending_rows)
        self._hop = int(engine.hop)
        if timed:
            self._time()
        self._group(groups, group_window)

    def arbitrate(self, multi, speech_samples: int = 12000, noise_samples: int = 8000) -> None:
        """StreamDetector.arbitrate for this detector: `multi` must be the engine it was made with, whose history the updates
        already read their clock from; ties below the level go to the lowest global stream.  The defaults are guesses."""
        if multi is not self.engine:
            raise ValueError("a models detector is arbitrated with the engine it was made with")
        self._arbitrate(multi, speech_samples, noise_samples)

    def set_groups(self, stream_ids, groups) -> None:
        """Put the listed GLOBAL streams in `groups` (one value or one per stream; -1: no group), for every WAKE model
        (mww_set_multi_detector_groups).  Ordered on the current CUDA stream; an open window keeps its candidates."""
        i, g = _group_list(stream_ids, groups, "stream_ids")
        self._check(self._L.mww_set_multi_detector_groups(self._d, i.ctypes.data, g.ctypes.data, i.size, self._cuda_stream()))

    @property
    def groups(self) -> np.ndarray:
        """int32 [n_streams]: every stream's group, -1 for none"""
        out = np.empty(self.engine.n_streams, np.int32)
        self._check(self._L.mww_get_multi_detector_groups(self._d, out.ctypes.data))
        return out

    @property
    def pending_rows(self) -> list:
        """each model's pending rows before the next call, as the detector will describe it"""
        return list(self._pending)

    def update(self, probs) -> None:
        """`probs`: what one engine call returned, one CUDA float32 tensor [members of model k, steps_k] per model (any row
        pitch; an OFF model's entry is not read and may be None).  Asynchronous on the current CUDA stream."""
        import torch
        K = self.n_models
        if len(probs) != K:
            raise ValueError("probs must hold one entry per model (%d)" % K)
        if any(not np.array_equal(a, b) for a, b in zip(self.streams, self.engine.streams)):
            raise ValueError("the engine's stream sets changed since this detector was made: make a new detector")
        ptrs, pitch, steps = (ctypes.c_void_p * K)(), (ctypes.c_longlong * K)(), (ctypes.c_int * K)()
        keep = []
        for k, p in enumerate(probs):
            if self.roles[k] == _lib.MWW_DETECT_OFF:
                continue
            rows = self.streams[k].size
            if (not isinstance(p, torch.Tensor) or not p.is_cuda or p.dtype != torch.float32 or p.dim() != 2 or p.shape[0] != rows
                    or p.device.index != self.device):
                raise ValueError("probs[%d] must be a CUDA float32 tensor [%d streams of model %d, steps] on device %d" % (k, rows, k, self.device))
            n = p.shape[1]
            if n and ((n > 1 and p.stride(1) != 1) or (rows > 1 and p.stride(0) < n)):
                p = p.contiguous()
            keep.append(p)
            ptrs[k] = p.data_ptr() if n and rows else None
            pitch[k] = p.stride(0) if rows > 1 else n
            steps[k] = n
        pend = (ctypes.c_int * K)(*self._pending)
        after = list(self.engine.pending_rows)
        if self.timed:
            S, b, hop = _history_clock(self.engine, None)
            if hop != self._hop:
                raise ValueError("the engine's hop changed since this detector was made (%d, was %d): make a new detector" % (hop, self._hop))
            self._check(self._L.mww_update_multi_detector_at(self._d, ptrs, pitch, steps, pend, (ctypes.c_int * K)(*after), S - b,
                                                             self._cuda_stream()))
        else:
            self._check(self._L.mww_multi_detector_update(self._d, ptrs, pitch, steps, pend, self._cuda_stream()))
        self._pending = after

    def drain(self):
        """-> (events, dropped): the events since the last drain (MODEL_EVENT_DTYPE, global stream ids) sorted by (model, step,
        stream), and how many more fired than `capacity` could hold.  Waits for the current CUDA stream; clears the event
        buffer and fired_ids."""
        return self._drain(MODEL_EVENT_DTYPE, ("model", "step", "stream"))

    def reset(self, stream_ids=None) -> None:
        """Fresh detector state of every model for all streams (None; the engine's pending rows are read again, so this is
        the call to make after engine.reset()) or the given GLOBAL stream ids: a host sequence, or a contiguous 1-D CUDA
        int32 tensor such as fired_ids.  Ids out of range are ignored."""
        self._reset(stream_ids, "stream ids")
        if stream_ids is None:
            self._pending = list(self.engine.pending_rows)

    def _used_model(self, k) -> int:
        if isinstance(k, bool) or not isinstance(k, (int, np.integer)) or not 0 <= int(k) < self.n_models:
            raise ValueError("k must be a model index in [0, %d)" % self.n_models)
        if self.roles[int(k)] == _lib.MWW_DETECT_OFF:
            raise ValueError("model %d is OFF: it has no rows" % int(k))
        return int(k)

    def set_cutoffs(self, k: int, stream_ids, cutoffs) -> None:
        """Give the listed GLOBAL streams of model k (WAKE or the VAD; members of its stream set) their own cutoffs
        (mww_set_multi_detector_cutoffs): `cutoffs` is one value or one per stream.  The first call switches every model to
        per-row mode, every other row keeping its model's cutoff.  Ordered on the current CUDA stream; the state and resets
        are unaffected."""
        k = self._used_model(k)
        ids, c = _cutoff_list(stream_ids, cutoffs, "stream_ids")
        self._check(self._L.mww_set_multi_detector_cutoffs(self._d, k, ids.ctypes.data, c.ctypes.data, ids.size, self._cuda_stream()))

    def get_cutoffs(self, k: int) -> np.ndarray:
        """float64 [members of model k]: each row's cutoff in the order of streams[k]"""
        k = self._used_model(k)
        out = np.empty(max(self.streams[k].size, 1), np.float64)
        self._check(self._L.mww_get_multi_detector_cutoffs(self._d, k, out.ctypes.data))
        return out[:self.streams[k].size]

    def _lookup(self, k) -> np.ndarray:
        """[n_streams]: the row of each global stream id in model k's list, -1 for a non-member (the lists are fixed)"""
        if not hasattr(self, "_inv"):
            self._inv = {}
        if k not in self._inv:
            inv = np.full(self.engine.n_streams, -1, np.int64)
            inv[self.streams[k]] = np.arange(self.streams[k].size)
            self._inv[k] = inv
        return self._inv[k]

    def export_streams(self, stream_ids) -> DetectorRecords:
        """Every model's row of the listed GLOBAL streams (hist, seen, cooldown or active) as packed records on this
        detector's device, ordered on the current CUDA stream in one launch (mww_export_detector_rows), with each stream's
        cutoff per model beside them (NaN where it is not a member).  A stream may be listed twice.  The detector does not
        change; events stay where they are (drain before moving)."""
        ids, data, layout = self._export(stream_ids, "stream_ids")
        cutoffs = []
        for k in range(self.n_models):
            c = np.full(ids.size, np.nan)
            if self.roles[k] != _lib.MWW_DETECT_OFF:
                row = self._lookup(k)[ids]
                c[row >= 0] = self.get_cutoffs(k)[row[row >= 0]]
            cutoffs.append(c)
        return DetectorRecords(data, layout, cutoffs)

    def import_streams(self, stream_ids, records: DetectorRecords) -> None:
        """Stream stream_ids[i] takes the rows records.data[i] holds (mww_import_detector_rows).  Per model: a stream that is
        not a member here ignores the record's slot; a member takes the slot's state, or fresh state (what reset gives) when
        the exported stream was not a member; every other stream is untouched.  A member whose exported cutoff differs from
        its own gets it (one set_cutoffs call per model, on the same CUDA stream).  After `engine.set_streams` this is how
        the stayers keep their rows: make a new detector and import every stream from the old one.  Records of another
        kind or rules, out-of-range or duplicate ids: MwwError with nothing changed; a malformed id list or records on
        another device: ValueError."""
        n = len(records.data)
        if records.layout.multi == 1 and records.layout.n_models == self.n_models:
            if len(records.cutoffs) != self.n_models or any(np.shape(c) != (n,) for c in records.cutoffs):
                raise ValueError("records.cutoffs must hold one cutoff per record for each of the %d models" % self.n_models)
        ids = self._import(stream_ids, records, "stream_ids")
        for k in range(self.n_models):
            if self.roles[k] == _lib.MWW_DETECT_OFF:
                continue
            row = self._lookup(k)[ids]
            c = np.asarray(records.cutoffs[k], np.float64)
            take = np.flatnonzero((row >= 0) & ~np.isnan(c))
            take = take[c[take] != self.get_cutoffs(k)[row[take]]]
            if take.size:
                self.set_cutoffs(k, ids[take], c[take])

    def _flag_name(self, k):
        return "active" if self.roles[k] == _lib.MWW_DETECT_VAD else "cooldown"

    def state_dict(self) -> dict:
        """{pending_rows: [p_k], models: [None for an OFF model, else {hist [n_k, window - 1], seen [n_k], cooldown or active [n_k]}]},
        and a grouped detector's groups [n_streams] and group_windows (GROUP_WINDOW_DTYPE [groups x WAKE models]), and an
        arbitrated one's group_levels (float32 [groups x WAKE models])"""
        models = []
        for k in range(self.n_models):
            if self.roles[k] == _lib.MWW_DETECT_OFF:
                models.append(None)
                continue
            n = self.streams[k].size
            m = {"hist": np.zeros((n, self.windows[k] - 1), np.float32), "seen": np.zeros(n, np.int64), self._flag_name(k): np.zeros(n, np.int32)}
            self._check(self._L.mww_multi_detector_get_state(self._d, k, m["hist"].ctypes.data, m["seen"].ctypes.data, m[self._flag_name(k)].ctypes.data))
            models.append(m)
        return self._group_state(dict(pending_rows=list(self._pending), models=models))

    def load_state_dict(self, d: dict) -> None:
        if len(d["models"]) != self.n_models or len(d["pending_rows"]) != self.n_models:
            raise ValueError("the state holds %d models, this detector %d" % (len(d["models"]), self.n_models))
        arrays = []
        for k, m in enumerate(d["models"]):
            if self.roles[k] == _lib.MWW_DETECT_OFF:
                arrays.append(None)
                continue
            if m is None:
                raise ValueError("model %d has no state" % k)
            n, flag = self.streams[k].size, self._flag_name(k)
            hist = np.ascontiguousarray(m["hist"], np.float32)
            seen = np.ascontiguousarray(m["seen"], np.int64)
            f = np.ascontiguousarray(m[flag], np.int32)
            if hist.shape != (n, self.windows[k] - 1) or seen.shape != (n,) or f.shape != (n,):
                raise ValueError("model %d: state must be hist [%d, window - 1], seen [%d], %s [%d]" % (k, n, n, flag, n))
            hi = 1 if self.roles[k] == _lib.MWW_DETECT_VAD else self.cooldown_slices[k]
            if (seen < 0).any() or (f < 0).any() or (f > hi).any():       # checked for every model before any is written
                raise ValueError("model %d: seen must not be negative and %s must be in [0, %d]" % (k, flag, hi))
            arrays.append((hist, seen, f))
        gw = self._load_group_state(d)
        for k, a in enumerate(arrays):
            if a is not None:
                self._check(self._L.mww_multi_detector_set_state(self._d, k, a[0].ctypes.data, a[1].ctypes.data, a[2].ctypes.data))
        self._apply_group_state(gw)
        self._pending = [int(p) for p in d["pending_rows"]]
