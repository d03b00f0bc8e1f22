"""Golden vectors for the streaming accuracy test of the reference's harness, produced by EXECUTING THE REFERENCE'S
OWN CODE: `compute_metrics`, `metrics_to_string` and `tflite_model_accuracy` are lifted out of
/root/reference/microwakeword/test.py with ast (the module cannot be imported: it imports TensorFlow at the top) and run
with stand-ins for `Model` (hands out seeded probability tracks in call order), `audio_processor` (get_data /
get_mode_duration), `os`, `open` (captures the metrics file) and `logging`.  Only inputs and outputs are stored.

    python tests/golden/make_accuracy_golden.py      (needs /root/reference; run in the authoring container)
"""

import ast
import json
import os
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference/microwakeword/test.py"
MIN_GAPS = (0, 3, 20)


def lifted(names, ns):
    tree = ast.parse(open(REF).read())
    nodes = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in names]
    exec(compile(ast.Module(body=nodes, type_ignores=[]), REF, "exec"), ns)
    return [ns[n] for n in names]


def tracks(rng, lengths):
    out = []
    for n in lengths:
        p = rng.beta(0.6, 0.9, n).astype(np.float32)
        p[rng.random(n) < 0.08] = np.float32(0.5)                     # the <= side of the crossing rule
        out.append(list(p))                                           # Model.predict_spectrogram returns a Python list
    return out


def run(data_set, probs, truth, min_gap, duration_s):
    written = {}

    class StubModel:
        def __init__(self, path):
            self.queue = list(probs)

        def predict_spectrogram(self, spectrogram):
            return self.queue.pop(0)

    class StubFile:
        def __init__(self, path):
            self.path = path

        def __enter__(self):
            return self

        def __exit__(self, *a):
            return False

        def write(self, s):
            written[self.path] = written.get(self.path, "") + s

    processor = types.SimpleNamespace(
        get_data=lambda mode, batch_size, features_length, truncation_strategy: (
            [np.zeros((len(p), 40), np.uint16) for p in probs], list(truth), None),
        get_mode_duration=lambda mode: duration_s)
    ns = {"np": np, "os": types.SimpleNamespace(path=os.path), "Model": StubModel,
          "logging": types.SimpleNamespace(info=lambda *a, **k: None), "open": lambda path, mode: StubFile(path)}
    compute_metrics, metrics_to_string, accuracy = lifted(["compute_metrics", "metrics_to_string", "tflite_model_accuracy"], ns)
    config = {"train_dir": "train", "batch_size": 1, "spectrogram_length": 204, "spectrogram_length_final_layer": min_gap}
    metrics = accuracy(config, "m", processor, data_set=data_set)
    (text,) = written.values()
    return metrics, text, compute_metrics, metrics_to_string


def main():
    rng = np.random.default_rng(2024)
    clip_lengths = [int(v) for v in rng.integers(1, 12, 60)] + [1, 2, 3]
    clips = tracks(rng, clip_lengths)
    truth = [bool(v) for v in rng.random(len(clips)) < 0.5]
    amb_lengths = [0, 1, 2, 3, 400, 37, 1000, 5, 260]
    amb = tracks(rng, amb_lengths)
    duration_s = 5400.0
    cases = []
    for min_gap in MIN_GAPS:
        for kind, probs, labels in (("testing", clips, truth), ("testing_ambient", amb, [False] * len(amb))):
            metrics, text, compute_metrics, metrics_to_string = run(kind, probs, labels, min_gap, duration_s)
            cases.append(dict(data_set=kind, min_gap=min_gap, metrics=metrics, text=text))
    # compute_metrics / metrics_to_string on their own, including the NaN branches
    extra = [(0.0, 0.0, 0.0, 0.0), (3.0, 0.0, 0.0, 0.0), (0.0, 4.0, 1.0, 0.0), (5.0, 7.0, 2.0, 1.0), (0.0, 0.0, 0.0, 9.0)]
    direct = [dict(args=a, metrics=compute_metrics(*a), text=metrics_to_string(compute_metrics(*a))) for a in extra]
    flat = lambda ts: np.asarray([v for t in ts for v in t], np.float32)
    np.savez(os.path.join(HERE, "accuracy_golden.npz"), clip_probs=flat(clips), clip_lengths=np.asarray(clip_lengths, np.int32),
             clip_truth=np.asarray(truth, bool), amb_probs=flat(amb), amb_lengths=np.asarray(amb_lengths, np.int32),
             duration_s=duration_s, cases=json.dumps(cases), direct=json.dumps(direct))
    for c in cases:
        print(c["data_set"], c["min_gap"], c["text"])


if __name__ == "__main__":
    main()
