"""oracle/accuracy_ref.py -- CPU ORACLE (test infrastructure) for the streaming accuracy test of the reference's
evaluation harness, microwakeword/test.py:406-517 (`tflite_model_accuracy`) and the helpers it reports with,
`compute_metrics` / `metrics_to_string` (test.py:30-91):

  * truncated sets (truncation_strategy != "none"): one prediction per clip, its LAST probability > 0.5
    (test.py:461-472); an empty probability list fails (probabilities[-1]);
  * ambient sets: per clip, previous probability and last positive index start at 0; a false accept is a step
    whose probability crosses 0.5 upwards (previous <= 0.5 < current) more than `min_gap`
    (config["spectrogram_length_final_layer"]) steps after the last counted one (test.py:473-484).

PARITY PINNED: tests/golden/accuracy_golden.npz was produced by executing the reference's own functions (lifted
with ast, see tests/golden/make_accuracy_golden.py); tests/test_batched_eval.py checks this restatement against it
exactly.  Kept apart from detection_ref.py so that file, pinned by its own golden, stays as it is.
"""

import numpy as np


def accuracy_track(probs, min_gap: int):
    """(false accepts of one ambient track, last probability > 0.5 or None for an empty track)."""
    p = [np.float32(v) for v in probs]
    count, last, prev = 0, 0, 0.0
    for j, v in enumerate(p):
        if prev <= 0.5 and v > 0.5 and j - last > min_gap:
            count += 1
            last = j
        prev = v
    return count, (bool(p[-1] > 0.5) if p else None)


def compute_metrics(tp, tn, fp, fn) -> dict:
    nan = float("nan")
    total = tp + tn + fp + fn
    out = dict(accuracy=nan, recall=nan, precision=nan, false_positive_rate=nan, false_negative_rate=nan, count=total)
    if total > 0:
        out["accuracy"] = (tp + tn) / total
    if fp + tn > 0:
        out["false_positive_rate"] = fp / (fp + tn)
    if tp + fn > 0:
        out["false_negative_rate"] = fn / (tp + fn)
        out["recall"] = tp / (tp + fn)
    if tp + fp > 0:
        out["precision"] = tp / (tp + fp)
    return out


def metrics_to_string(m: dict) -> str:
    pct = lambda v: format(v, ".4%")
    return "accuracy = %s; recall = %s; precision = %s; fpr = %s; fnr = %s; (N=%s)" % (
        pct(m["accuracy"]), pct(m["recall"]), pct(m["precision"]), pct(m["false_positive_rate"]), pct(m["false_negative_rate"]), m["count"])


def tflite_model_accuracy(prob_tracks, ground_truth, ambient: bool, min_gap: int, ambient_duration_s=None):
    """The metric side of test.py:406-517 on per-clip probability lists -> (metrics dict, metrics string)."""
    tp = tn = fp = fn = 0.0
    for probs, truth in zip(prob_tracks, ground_truth):
        count, last_positive = accuracy_track(probs, min_gap)
        if ambient:
            fp += count
            continue
        if last_positive is None:
            raise IndexError("list index out of range")
        if truth == last_positive:
            if truth:
                tp += 1
            else:
                tn += 1
        elif truth:
            fn += 1
        else:
            fp += 1
    m = compute_metrics(tp, tn, fp, fn)
    if ambient:
        return m, "false accepts = {}; false accepts per hour = {:.4}".format(fp, fp / (ambient_duration_s / 3600.0))
    return m, metrics_to_string(m)
