"""Time of the hybrid kernel (fp32 graph with int8-weight ops, nn_generic_hybrid_kernel) at 65 536 streams, against the
same weights as fp32 on the generic kernel (MWW_FORCE_GENERIC=1) and on the default (compiled-in okay_nabu) kernels:
  * a 3 s predict_clip call;
  * a 480-sample live step() call;
  * Model.predict_spectrograms over the tools/eval_time.py workload (`clips` 204-row tracks + `hours` one-hour tracks).
Hybrid okay_nabu: okay_nabu_synth_f32.mww written as a float .tflite whose >= 1024-element kernels are per-channel int8
(the converter's dynamic-range rule); fp32 arms: the dequantised weights as float32.  Arms alternate over the rounds.
Prints the card and its power limit read in the same run.
    python tools/hybrid_time.py [clips] [hours]"""
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import tflite_hybrid_writer as HW  # noqa: E402
from microwakeword_b200 import model_file as MF  # noqa: E402
from microwakeword_b200 import tflite_file as TF  # noqa: E402
from microwakeword_b200.engine import StreamEngine  # noqa: E402
from microwakeword_b200.inference import Model  # noqa: E402

CLIPS = int(sys.argv[1]) if len(sys.argv) > 1 else 10000
HOURS = int(sys.argv[2]) if len(sys.argv) > 2 else 4
ROUNDS = 3
S = 65536


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "%s (nvidia-smi unavailable)" % torch.cuda.get_device_name(0)


def timed(fn, reps=1):
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) / reps


def make_engine(blob, generic):
    if generic:
        os.environ["MWW_FORCE_GENERIC"] = "1"
    try:
        return StreamEngine(blob, n_streams=S)
    finally:
        os.environ.pop("MWW_FORCE_GENERIC", None)


def make_model(blob, generic):
    if generic:
        os.environ["MWW_FORCE_GENERIC"] = "1"
    try:
        return Model(blob)
    finally:
        os.environ.pop("MWW_FORCE_GENERIC", None)


def main():
    f32 = MF.load(os.path.join(ROOT, "tests", "golden", "okay_nabu_synth_f32.mww"))
    hy = TF.tensors_from_tflite(HW.write_hybrid_mixednet(f32, lambda op, n: n >= 1024))
    arms = {"hybrid": (MF.write_container(hy), False),
            "fp32_generic": (MF.write_container({k: v for k, v in hy.items() if not k.startswith("hy/")}), True),
            "fp32_default": (MF.write_container({k: v for k, v in hy.items() if not k.startswith("hy/")}), False)}
    print("card:", card())
    g = torch.Generator(device="cuda").manual_seed(1)
    clip = torch.randint(-4000, 4000, (S, 48000), device="cuda", dtype=torch.int16, generator=g)
    live = clip[:, :480].contiguous()
    res = {k: {"clip": [], "live": [], "spectrograms": []} for k in arms}
    engines = {k: make_engine(b, gen) for k, (b, gen) in arms.items()}
    for r in range(ROUNDS):
        for k, eng in engines.items():
            eng.reset()
            res[k]["clip"].append(timed(lambda: eng.predict_clip(clip)))
            eng.reset()
            eng.step(live)
            res[k]["live"].append(timed(lambda: eng.step(live), reps=10))
    del engines, clip, live
    torch.cuda.empty_cache()
    rng = np.random.default_rng(0)
    tracks = [rng.integers(0, 1000, (204, 40)).astype(np.uint16) for _ in range(CLIPS)]
    tracks += [rng.integers(0, 1000, (360000, 40)).astype(np.uint16) for _ in range(HOURS)]
    models = {k: make_model(b, gen) for k, (b, gen) in arms.items()}
    for r in range(ROUNDS - 1):
        for k, m in models.items():
            m.engine.reset()
            res[k]["spectrograms"].append(timed(lambda: m.predict_spectrograms(tracks)))
    for k in arms:
        print("%-13s clip 3 s: %8.2f ms   live 480: %7.3f ms   predict_spectrograms (%d clips + %d h): %8.1f ms" % (
            k, 1e3 * min(res[k]["clip"]), 1e3 * min(res[k]["live"]), CLIPS, HOURS, 1e3 * min(res[k]["spectrograms"])))
    print("card:", card())


if __name__ == "__main__":
    main()
