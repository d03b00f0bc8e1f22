#!/usr/bin/env python
"""Where a stream's cycles go in the wgmma clip kernel (nn_f32_clip_tc_kernel): builds an instrumented copy of the library with
-DMWW_TC_PHASE_CLOCKS into a temporary directory, runs the benchmark's clip shape (65 536 streams x 3 s, fp32 model) and prints the
mean clock64() cycles per stream per phase, as seen by thread 0 of each CTA (a CTA's timeline: it waits at every CTA-wide barrier).
The counters add a few instructions and atomics per phase edge, so the kernel time printed here is that of the instrumented build.
    python tools/tc_phases.py [calls]"""
import atexit
import ctypes
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

# the first conv builds its A operand in registers, inside its MMA phase; "produce: first-conv A" is left for kernels that stage it in
# shared memory (the phase edges are the same in every version of the kernel, so two versions' tables compare row by row)
PHASES = ["stream start", "feature-rows wait", "produce: first-conv A", "produce: depthwise", "publish (weights wait, fence, barrier)",
          "MMA: first conv", "MMA: 1x1 projections", "release (barrier, next weights)", "block end: x_to_ring", "block end: ring_to_x",
          "block end: epilogue", "head", "call end (first-conv ring, pending rows)"]

calls = int(sys.argv[1]) if len(sys.argv) > 1 else 10
S = int(os.environ.get("TC_PHASE_STREAMS", "65536"))
tmp = tempfile.mkdtemp(prefix="mww_tc_phases_")
atexit.register(shutil.rmtree, tmp, True)
so = os.path.join(tmp, "libmww_b200_phases.so")
cmd = [build.NVCC] + build.FLAGS + ["-DMWW_TC_PHASE_CLOCKS", "-o", so] + [os.path.join(build.CSRC, s) for s in build.SOURCES]
res = subprocess.run(cmd, capture_output=True, text=True)
if res.returncode != 0:
    sys.exit(res.stdout + res.stderr)
_lib.SO_PATH = so                              # the engine binds this copy in place of the product library
from microwakeword_b200.engine import StreamEngine  # noqa: E402

L = _lib.lib()
L.mww_tc_phase_read.restype = ctypes.c_int
L.mww_tc_phase_read.argtypes = [ctypes.c_void_p, ctypes.c_int]
counters = (ctypes.c_ulonglong * (len(PHASES) + 1))()

dev = torch.device("cuda", 0)
eng = StreamEngine(model_blob("f32"), n_streams=S, device=0)
audio = synth_audio_device(torch, S, 48000, 1, dev)
for _ in range(2):
    eng.predict_clip(audio)
torch.cuda.synchronize()
assert L.mww_tc_phase_read(counters, 1) == 0
eng.profile(True)
for _ in range(calls):
    eng.predict_clip(audio)
torch.cuda.synchronize()
assert L.mww_tc_phase_read(counters, 1) == 0
prof = eng.profile_read()
streams = counters[len(PHASES)]
assert streams == S * calls, (streams, S * calls)
total = sum(counters[i] for i in range(len(PHASES)))
name = torch.cuda.get_device_name(0)
smi = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip()
print("%s (%s); %d streams x %d calls; instrumented mixednet %.2f ms per call" % (name, smi, S, calls,
      prof["mixednet"][0] / max(prof["mixednet"][1], 1)))
print("%-44s %12s %7s" % ("phase (thread 0 of each CTA)", "cycles/stream", "share"))
for i, p in enumerate(PHASES):
    print("%-44s %12.0f %6.1f%%" % (p, counters[i] / streams, 100.0 * counters[i] / max(total, 1)))
print("%-44s %12.0f" % ("total", total / streams))
