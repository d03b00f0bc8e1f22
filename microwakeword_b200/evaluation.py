"""Non-streaming batched evaluation around the clip kernel (SURVEY.md section 8 row f-4): the data side of
``microwakeword.data.FeatureHandler.get_data(..., truncation_strategy="split")`` (data.py:301-311) and the metric
bookkeeping of ``microwakeword.train.validate_nonstreaming`` (train.py:41-163), with ``model.evaluate(batch_size=1024)``
replaced by ``Model.predict_nonstreaming`` (the GPU clip kernel evaluated on whole windows).

Streaming accuracy (``microwakeword.test.tflite_model_accuracy``, test.py:406-517, with ``compute_metrics`` and
``metrics_to_string`` of test.py:30-91): ``tflite_model_accuracy`` below, on the batched state-carrying pass of
``Model.predict_spectrograms`` and the accuracy kernel of csrc/mww_detect.cu.

Training itself (train.py:166-), the Keras metric objects and the feature store are out of scope; these functions take
plain arrays so the reference's harness can call them with what it already has."""

from __future__ import annotations

import numpy as np

from .model_file import FEATURE_SCALE


def split_ambient(spectrogram: np.ndarray, features_length: int, step_s: float = 0.01, stride: int = 3):
    """data.py:297-311, truncation_strategy == "split": windows of `features_length` rows starting every
    int(1000 * step * stride) rows (30 rows = 300 ms for the 10 ms / stride-3 models), for start in
    range(0, T - features_length, hop) -- so a window that would end exactly at the last row is NOT produced.
    uint16 spectrograms are scaled by 0.0390625 first (data.py:297-298).  Returns float32 [n, features_length, 40]."""
    spec = np.asarray(spectrogram)
    if np.issubdtype(spec.dtype, np.uint16):
        spec = spec.astype(np.float32) * np.float32(FEATURE_SCALE)
    hop = int(1000 * step_s * stride)
    if hop < 1:
        raise ValueError("range() arg 3 must not be zero")          # what the reference's range() raises
    starts = range(0, spec.shape[0] - features_length, hop)
    if len(starts) == 0:
        return np.zeros((0, features_length, spec.shape[1]), np.float32)
    return np.stack([spec[s:s + features_length] for s in starts]).astype(np.float32, copy=False)


def threshold_counts(predictions, labels, cutoffs=None):
    """What the Keras TruePositives / FalsePositives / FalseNegatives metrics hold for thresholds np.linspace(0, 1, 101)
    (train.py:44-56): a prediction is positive when it is strictly greater than the threshold."""
    cut = np.linspace(0.0, 1.0, 101) if cutoffs is None else np.asarray(cutoffs, np.float64)
    p = np.asarray(predictions, np.float32).reshape(-1).astype(np.float64)
    y = np.asarray(labels).reshape(-1).astype(bool)
    pos = p[None, :] > cut[:, None]
    return dict(tp=(pos & y[None, :]).sum(1).astype(np.float64), fp=(pos & ~y[None, :]).sum(1).astype(np.float64),
                fn=(~pos & y[None, :]).sum(1).astype(np.float64), cutoffs=cut)


def viable_recall_metrics(tp, fp_ambient, fn, ambient_duration_h: float) -> dict:
    """train.py:99-161: recall / false accepts per hour per cutoff, the cutoff with no false accepts, and the average recall
    over 0..2 false accepts per hour (trapezoid of the recall-vs-faph curve, interpolated at 2 faph, divided by 2)."""
    tp, fp, fn = (np.asarray(v, np.float64) for v in (tp, fp_ambient, fn))
    recall = tp / (tp + fn)
    faph = fp / ambient_duration_h
    cutoffs = np.linspace(0.0, 1.0, 101)
    cutoff_no_faph, recall_no_faph = 1.0, None
    for i, c in enumerate(cutoffs):
        if faph[i] == 0:
            cutoff_no_faph, recall_no_faph = c, recall[i]
            break
    if recall_no_faph is None:
        raise UnboundLocalError("no cutoff reaches 0 false accepts per hour (the reference fails here as well, train.py:158)")
    if faph[0] > 2:
        k = 1
        while faph[k] > 2:
            k += 1
        x0, y0, x1, y1 = faph[k - 1], recall[k - 1], faph[k], recall[k]
        first = (y0 * (x1 - 2.0) + y1 * (2.0 - x0)) / (x1 - x0)
    else:
        k, first = 0, recall[0]
    xs, ys = [2.0], [first]
    for i in range(k, len(recall)):
        if faph[i] != xs[-1]:
            xs.append(faph[i])
            ys.append(recall[i])
    x, y = np.asarray(xs[::-1]), np.asarray(ys[::-1])
    average = float(np.sum((x[1:] - x[:-1]) * (y[1:] + y[:-1]) / 2.0)) / 2.0
    return dict(recall_at_no_faph=recall_no_faph, cutoff_for_no_faph=cutoff_no_faph, ambient_false_positives=fp[50],
                ambient_false_positives_per_hour=faph[50], average_viable_recall=average)


def validate_nonstreaming(model, test_fingerprints, test_ground_truth, ambient_spectrograms=None, ambient_duration_h: float = 0.0,
                          features_length: int | None = None, step_s: float = 0.01, stride: int = 3, batch_size: int = 1024) -> dict:
    """train.py:41-163 on arrays: `test_fingerprints` [n, features_length, 40] with boolean labels, and (optionally) the
    ambient set as a list of long spectrograms that is split like data.py:301-311.  Accuracy / recall / precision come from
    the 0.5 threshold (Keras defaults); auc and loss are Keras-internal and not reproduced."""
    features_length = features_length or model.nonstreaming_length()
    probs = model.predict_nonstreaming(np.asarray(test_fingerprints), batch_size=batch_size)
    counts = threshold_counts(probs, test_ground_truth)
    y = np.asarray(test_ground_truth).reshape(-1).astype(bool)
    tp, fp, fn = counts["tp"][50], counts["fp"][50], counts["fn"][50]
    tn = float((~y).sum()) - fp
    metrics = dict(accuracy=(tp + tn) / max(len(y), 1), recall=tp / max(tp + fn, 1.0), precision=tp / max(tp + fp, 1.0),
                   recall_at_no_faph=0, cutoff_for_no_faph=0, ambient_false_positives=0, ambient_false_positives_per_hour=0,
                   average_viable_recall=0)
    if ambient_spectrograms:
        windows = [split_ambient(sp, features_length, step_s, stride) for sp in ambient_spectrograms]
        windows = np.concatenate([w for w in windows if len(w)], 0)
        amb = threshold_counts(model.predict_nonstreaming(windows, batch_size=batch_size), np.zeros(len(windows), bool))
        # the reference accumulates both sets in one metric object and subtracts the test set's false positives (:95-97)
        metrics.update(viable_recall_metrics(counts["tp"], amb["fp"], counts["fn"], ambient_duration_h))
    return metrics


def compute_metrics(true_positives, true_negatives, false_positives, false_negatives) -> dict:
    """Drop-in for microwakeword.test.compute_metrics (test.py:30-73): accuracy, recall, precision, false positive and
    false negative rates and the sample count; a rate whose denominator is 0 is NaN."""
    tp, tn, fp, fn = true_positives, true_negatives, false_positives, false_negatives
    nan = float("nan")
    count = tp + tn + fp + fn
    has_pos, has_neg = tp + fn > 0, fp + tn > 0
    return {
        "accuracy": (tp + tn) / count if count > 0 else nan,
        "recall": tp / (tp + fn) if has_pos else nan,
        "precision": tp / (tp + fp) if tp + fp > 0 else nan,
        "false_positive_rate": fp / (fp + tn) if has_neg else nan,
        "false_negative_rate": fn / (tp + fn) if has_pos else nan,
        "count": count,
    }


def metrics_to_string(metrics: dict) -> str:
    """Drop-in for microwakeword.test.metrics_to_string (test.py:76-91): rates as percentages with 4 decimals."""
    rates = [("accuracy", "accuracy"), ("recall", "recall"), ("precision", "precision"), ("fpr", "false_positive_rate"),
             ("fnr", "false_negative_rate")]
    return "; ".join("%s = %s" % (label, format(metrics[key], ".4%")) for label, key in rates) + "; (N=%s)" % (metrics["count"],)


def _chunk_count(model, n_rows: int) -> int:
    """Steps predict_spectrogram runs on a track of n_rows rows (inference.py:98-105)."""
    return len(range(model.input_feature_slices, n_rows + 1, model.stride))


def tflite_model_accuracy(model, fingerprints, ground_truth, ambient: bool, spectrogram_length_final_layer: int,
                          ambient_duration_s: float | None = None):
    """microwakeword.test.tflite_model_accuracy (test.py:406-517) on arrays: the spectrograms the reference's
    ``audio_processor.get_data`` returns, their labels, and whether the set is an ambient one (``data_set`` ending in
    "ambient", truncation strategy "none").  Returns (metrics dict, metrics string) -- the dict the reference returns and
    the string it logs and writes to its accuracy file.

    Every fingerprint is cast to float32 (test.py:447; uint16 features are therefore NOT scaled by 0.0390625 here) and
    fed to one model in order with the state carried over, as the reference does; a microwakeword_b200 Model does this
    as one batched pass (Model.predict_spectrograms) and the per-track rule runs on the GPU (detection.accuracy_counts).
      * ambient=False: each track is one prediction, its last probability > 0.5, against its label.  A track too short
        for one model step raises IndexError, as ``probabilities[-1]`` does in the reference.  For a model that has
        ``input_feature_slices`` and ``stride`` (a Model), only the tracks up to that one are fed, as in the reference;
        any other model object has been fed every track when the error is raised.
      * ambient=True: false accepts are rising crossings of 0.5 (previous <= 0.5 < current), counted only when more
        than spectrogram_length_final_layer steps after the last counted one; the previous probability and the last
        index restart at 0 on every track, so crossings in a track's first spectrogram_length_final_layer steps are never
        counted.  The string gives false accepts per hour over ambient_duration_s (audio_processor.get_mode_duration).
    An empty set fails as the reference does (its metrics are never assigned)."""
    from . import detection
    fps = [np.asarray(f).astype(np.float32) for f in fingerprints]
    if not fps:
        raise UnboundLocalError("tflite_model_accuracy: no fingerprints (the reference's metrics are never assigned)")
    if ambient and ambient_duration_s is None:
        raise ValueError("tflite_model_accuracy: an ambient set needs ambient_duration_s")
    if not ambient and hasattr(model, "input_feature_slices") and hasattr(model, "stride"):
        empty = next((i for i, f in enumerate(fps) if _chunk_count(model, f.shape[0] if f.ndim else 0) == 0), None)
        if empty is not None:
            fps = fps[:empty + 1]                       # the reference stops at this track
    device = getattr(getattr(model, "engine", None), "device", 0)
    probs = detection.model_probabilities(model, fps, device)
    lengths = probs.lengths if isinstance(probs, detection._Packed) else [len(p) for p in probs]
    empty = next((i for i, n in enumerate(lengths) if n == 0), None)
    if not ambient and empty is not None:
        raise IndexError("list index out of range (track %d gives no probabilities: probabilities[-1])" % empty)
    false_accepts, last_positive = detection.accuracy_counts(probs, spectrogram_length_final_layer, device)
    tp = tn = fp = fn = 0.0
    if ambient:
        fp = float(false_accepts.sum())
        metrics = compute_metrics(tp, tn, fp, fn)
        return metrics, "false accepts = {}; false accepts per hour = {:.4}".format(fp, fp / (ambient_duration_s / 3600.0))
    truth = np.asarray(ground_truth).reshape(-1)[:len(fps)]
    hit = truth == last_positive                                    # sample_ground_truth == prediction
    positive = truth.astype(bool)                                   # if sample_ground_truth
    tp, tn = float((hit & positive).sum()), float((hit & ~positive).sum())
    fn, fp = float((~hit & positive).sum()), float((~hit & ~positive).sum())
    metrics = compute_metrics(tp, tn, fp, fn)
    return metrics, metrics_to_string(metrics)
