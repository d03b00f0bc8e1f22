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
"""

from __future__ import annotations

import ctypes

import numpy as np

from . import _lib


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
