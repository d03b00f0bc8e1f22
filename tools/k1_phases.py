#!/usr/bin/env python
"""Where a stream's cycles go in the fused clip frontend (k1_clip_kernel): builds an instrumented copy of its companion
library with -DMWW_K1_PHASE_CLOCKS, and a libmww_b200.so that links it, into a temporary directory, runs the benchmark's clip shape
(65 536 streams x 3 s, fp32 model) and prints the mean clock64() cycles per stream per phase, as seen by thread 0 of each CTA (a
CTA's timeline: it runs the estimate chain and waits at every CTA-wide barrier; one CTA per stream).  "stream start" is the table
staging, the estimate load and the first group's load.  The counters add a few instructions and atomics per phase edge, so the
kernel time printed here is that of the instrumented build.
    python tools/k1_phases.py [calls]"""
import atexit
import ctypes
import glob
import os
import shutil
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import model_blob, synth_audio_device  # noqa: E402
from microwakeword_b200 import _lib, build  # noqa: E402

PHASES = ["stream start (tables, estimate, audio)", "top barrier (audio wait)", "prefetch issue", "pass 1: window, FFT stages 1-2",
          "pass 2: FFT stages 3-4", "real-FFT post-pass, |X|^2", "filterbank, sqrt", "filterbank barrier", "estimate chain + barrier",
          "outputs: noise, PCAN, log"]

calls = int(sys.argv[1]) if len(sys.argv) > 1 else 10
S = int(os.environ.get("K1_PHASE_STREAMS", "65536"))
build.build()
tmp = tempfile.mkdtemp(prefix="mww_k1_phases_")
atexit.register(shutil.rmtree, tmp, True)
# every companion library as built, then the instrumented frontend library over its copy, then a main library linked against them
# (rpath $ORIGIN: the temporary directory)
companions = [p for p in glob.glob(os.path.join(build.HERE, "libmww_*.so")) if p != build.OUT]
for p in companions:
    shutil.copy(p, tmp)


def nvcc(out, sources, extra):
    res = subprocess.run([build.NVCC] + build.FLAGS + ["-o", out] + [os.path.join(build.CSRC, s) for s in sources] + extra,
                         capture_output=True, text=True)
    if res.returncode != 0:
        sys.exit(res.stdout + res.stderr)


nvcc(os.path.join(tmp, os.path.basename(build.FC_OUT)), build.FC_SOURCES, ["-DMWW_K1_PHASE_CLOCKS"])
so = os.path.join(tmp, "libmww_b200.so")
nvcc(so, build.SOURCES, ["-L" + tmp] + ["-l" + os.path.basename(p)[3:-3] for p in companions] + ["-Xlinker", "-rpath,$ORIGIN"])
_lib.SO_PATH = so                              # the engine binds this copy in place of the product library
from microwakeword_b200.engine import StreamEngine  # noqa: E402

L = _lib.lib()
L.mww_k1_phase_read.restype = ctypes.c_int
L.mww_k1_phase_read.argtypes = [ctypes.c_void_p, ctypes.c_int]
counters = (ctypes.c_ulonglong * (len(PHASES) + 1))()

dev = torch.device("cuda", 0)
eng = StreamEngine(model_blob("f32"), n_streams=S, device=0)
audio = synth_audio_device(torch, S, 48000, 1, dev)
for _ in range(2):
    eng.predict_clip(audio)
torch.cuda.synchronize()
assert L.mww_k1_phase_read(counters, 1) == 0
eng.profile(True)
for _ in range(calls):
    eng.predict_clip(audio)
torch.cuda.synchronize()
assert L.mww_k1_phase_read(counters, 1) == 0
prof = eng.profile_read()
streams = counters[len(PHASES)]
assert streams == S * calls, (streams, S * calls)
total = sum(counters[i] for i in range(len(PHASES)))
name = torch.cuda.get_device_name(0)
smi = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip()
print("%s (%s); %d streams x %d calls; instrumented k1_spectral %.2f ms per call" % (name, smi, S, calls,
      prof["k1_spectral"][0] / max(prof["k1_spectral"][1], 1)))
print("%-44s %12s %7s" % ("phase (thread 0 of each CTA)", "cycles/stream", "share"))
for i, p in enumerate(PHASES):
    print("%-44s %12.0f %6.1f%%" % (p, counters[i] / streams, 100.0 * counters[i] / max(total, 1)))
print("%-44s %12.0f" % ("total", total / streams))
