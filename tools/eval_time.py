"""What the batched evaluation pass saves: the reference's per-track loop (Model.predict_spectrogram once per track, state
carried) against Model.predict_spectrograms (one batched pass, same results), and detection.streaming_model_roc both
ways (a model object that only has predict_spectrogram takes the per-track loop).  Synthetic test set: `clips` tracks of
204 rows (positive-clip sized) plus `hours` one-hour ambient tracks (360 000 rows each), uint16 features.  int8 and fp32
okay_nabu; the two sides alternate over two rounds, every side starting from a reset model; the probabilities of the two
sides are compared (int8 exact, fp32 within 1e-5).  Also times detection.accuracy_counts (mww_accuracy_counts plus its
host copies) on the ambient probabilities alone, five calls.  Prints the card and its power limit read in the same run.
    python tools/eval_time.py [clips] [hours]"""
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from microwakeword_b200 import detection  # noqa: E402
from microwakeword_b200.inference import Model  # noqa: E402

CLIPS = int(sys.argv[1]) if len(sys.argv) > 1 else 10000
HOURS = int(sys.argv[2]) if len(sys.argv) > 2 else 4
ROUNDS = 2
GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "%s (nvidia-smi unavailable)" % torch.cuda.get_device_name(0)


class LoopOnly:
    """An object with nothing but predict_spectrogram: streaming_model_roc runs its per-track loop on it."""

    def __init__(self, model):
        self.predict_spectrogram = model.predict_spectrogram


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t, out


def main():
    rng = np.random.default_rng(5)
    feats = np.load(os.path.join(GOLDEN, "config0_features.npy"))          # uint16 [997, 40] of real frontend output
    pick = lambda n: feats[rng.integers(0, feats.shape[0], n)]             # rows drawn from it: realistic value ranges
    ambient = [pick(360000) for _ in range(HOURS)]
    clips = [pick(204) for _ in range(CLIPS)]
    tracks = ambient + clips
    print("card: %s" % card())
    print("test set: %d clips x 204 rows + %d x 1 h ambient = %d tracks, %d rows" % (CLIPS, HOURS, len(tracks), sum(t.shape[0] for t in tracks)))
    for kind in ("int8", "f32"):
        m = Model(os.path.join(GOLDEN, "okay_nabu_synth_%s.mww" % kind))
        warm = [ambient[0][:30000]] + clips[:300] if ambient else clips[:300]   # warm-up: module load, engines, staging buffer
        m.reset()
        [m.predict_spectrogram(t) for t in warm]
        m.reset()
        m.predict_spectrograms(warm)
        times = {k: [] for k in ("loop", "batched", "roc_loop", "roc_batched")}
        for r in range(ROUNDS):
            m.reset()
            dt, want = timed(lambda: [m.predict_spectrogram(t) for t in tracks])
            times["loop"].append(dt)
            m.reset()
            dt, got = timed(lambda: m.predict_spectrograms(tracks))
            times["batched"].append(dt)
            w, g = np.concatenate([np.asarray(x, np.float32) for x in want]), np.concatenate([np.asarray(x, np.float32) for x in got])
            err = float(np.abs(w - g).max())
            assert w.shape == g.shape and (err == 0.0 if kind == "int8" else err <= 1e-5), (kind, err)
            m.reset()
            dt, roc_a = timed(lambda: detection.streaming_model_roc(LoopOnly(m), ambient, clips))
            times["roc_loop"].append(dt)
            m.reset()
            dt, roc_b = timed(lambda: detection.streaming_model_roc(m, ambient, clips))
            times["roc_batched"].append(dt)
            if kind == "int8":
                assert np.array_equal(roc_a["faph"], roc_b["faph"]) and np.array_equal(roc_a["frr"], roc_b["frr"])
        m.reset()
        packed = detection.model_probabilities(m, ambient)                  # the ambient probabilities, left on the GPU
        detection.accuracy_counts(packed, 20)
        acc = [timed(lambda: detection.accuracy_counts(packed, 20))[0] for _ in range(5)]
        times["accuracy_kernel_ambient"] = acc
        steps = int(g.size)
        print("%s: %d steps; max |loop - batched| = %.3g" % (kind, steps, err))
        for k, v in times.items():
            print("  %-24s %s s" % (k, "  ".join("%.4f" % x for x in v)))
        print("  speed-up    predict: %.1fx   roc: %.1fx" % (min(times["loop"]) / min(times["batched"]), min(times["roc_loop"]) / min(times["roc_batched"])))


if __name__ == "__main__":
    main()
