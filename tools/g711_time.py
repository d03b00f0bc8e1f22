"""What G.711 input saves: the same calls with int16 and with mu-law audio at --streams (65 536 by default), two engines fed
the same samples (the int16 arm gets the decoded codes), alternating inside each round; their probabilities and features
must be bit-identical (checked).

  (a) host clip ... an 8 kHz handle, 3 s calls (24 000 samples) from pinned host memory: predict_clip_host with int16 against
                    mu-law.  The host path is PCIe-bound, so the bytes a call copies (printed beside the time) decide it.
  (b) host live ... the same handles, 240-sample live calls (30 ms at 8 kHz) from pinned host memory.
  (c) device clip . a 16 kHz frontend-only handle, 3 s calls (48 000 samples) already on the device: features with int16
                    against mu-law, CUDA events around the call.  This is the decode's cost inside the compute-bound clip
                    kernel.
Times in ms per call (host wall clock around the synchronous host calls; device events for (c)), one figure per round.
Prints the card, its power limit and the SM clock sampled during the run.  There is no CPU path: without a GPU it fails.
    python tools/g711_time.py [--streams 65536] [--rounds 3] [--clip-calls 3] [--live-calls 50]"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import ClockSampler, model_blob, synth_audio_device  # noqa: E402
from microwakeword_b200.engine import StreamEngine, host_array  # noqa: E402

P = 1021                         # distinct base streams; stream s carries base[s % P]


def ulaw_table():
    """int16 [256]: the mu-law decode of include/mww.h"""
    u = (~np.arange(256)) & 0xFF
    t = (((u & 0x0F) << 3) + 0x84) << ((u & 0x70) >> 4)
    return np.where(u & 0x80, 0x84 - t, t - 0x84).astype(np.int16)


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "%s (nvidia-smi unavailable)" % torch.cuda.get_device_name(0)


def codes_for(n, seed):
    """uint8 [P, n] mu-law codes of the benchmark's synthetic audio (the code whose value is the first >= the sample), and
    their decoded int16 samples"""
    table = ulaw_table()
    order = np.argsort(table, kind="stable")
    x = synth_audio_device(torch, P, n, seed, torch.device("cuda", 0)).cpu().numpy()
    pos = np.minimum(np.searchsorted(table[order], x), 255)
    codes = order[pos].astype(np.uint8)
    return codes, table[codes]


def tiled(base, S, dtype, pinned):
    out = host_array((S, base.shape[1]), dtype) if pinned else np.empty((S, base.shape[1]), dtype)
    for s0 in range(0, S, P):
        out[s0:s0 + P] = base[:min(P, S - s0)]
    return out


def host_arms(S, n, calls, rounds):
    """(a) / (b): -> {arm: [ms per call per round]}, bytes copied per call per arm"""
    codes, pcm = codes_for(n, 7)
    audio = {"int16": tiled(pcm, S, np.int16, True), "ulaw": tiled(codes, S, np.uint8, True)}
    blob = model_blob("f32")
    eng = {k: StreamEngine(blob, n_streams=S, input_rate=8000) for k in audio}
    outs = {k: host_array((S, 128), np.float32) for k in audio}
    run = {"int16": lambda: eng["int16"].predict_clip_host(audio["int16"], out=outs["int16"]),
           "ulaw": lambda: eng["ulaw"].predict_clip_host(audio["ulaw"], out=outs["ulaw"], law="ulaw")}
    last = {}
    for k in audio:                              # warm-up: module load, staging buffers, a steady buffered count
        for _ in range(2):
            last[k] = run[k]()
    times = {k: [] for k in audio}
    for _ in range(rounds):
        for k in audio:
            t0 = time.perf_counter()
            for _ in range(calls):
                last[k] = run[k]()
            times[k].append((time.perf_counter() - t0) * 1e3 / calls)
    assert last["int16"].shape == last["ulaw"].shape and np.array_equal(last["int16"].view(np.int32), last["ulaw"].view(np.int32))
    for e in eng.values():
        e.close()
    return times, {k: a.nbytes for k, a in audio.items()}


def device_arms(S, n, calls, rounds):
    """(c): -> {arm: [ms per call per round]} of features on device-resident audio"""
    codes, pcm = codes_for(n, 9)
    idx = torch.arange(S, device="cuda") % P
    audio = {"int16": torch.from_numpy(pcm).cuda()[idx], "ulaw": torch.from_numpy(codes).cuda()[idx]}
    eng = {k: StreamEngine(None, n_streams=S) for k in audio}
    law = {"int16": None, "ulaw": "ulaw"}
    last = {}
    for k in audio:
        for _ in range(2):
            last[k] = eng[k].features(audio[k], law=law[k])
    times = {k: [] for k in audio}
    for _ in range(rounds):
        for k in audio:
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            for _ in range(calls):
                last[k] = eng[k].features(audio[k], law=law[k])
            end.record()
            end.synchronize()
            times[k].append(start.elapsed_time(end) / calls)
    assert torch.equal(last["int16"].view(torch.int16), last["ulaw"].view(torch.int16))
    for e in eng.values():
        e.close()
    return times


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--streams", type=int, default=65536)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--clip-calls", type=int, default=3)
    ap.add_argument("--live-calls", type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("g711_time.py measures the GPU kernels and needs a CUDA device; none is available")
    S = a.streams
    print("card: %s; %d streams, fp32 okay_nabu, pinned host audio" % (card(), S))
    clocks = ClockSampler(0)
    try:
        clip = host_arms(S, 24000, a.clip_calls, a.rounds)
        live = host_arms(S, 240, a.live_calls, a.rounds)
        dev = device_arms(S, 48000, a.clip_calls, a.rounds)
    finally:
        sampled = clocks.stop()
    print("SM clock during the run: median %s MHz (max %s MHz), throttle reasons seen: %s" %
          (sampled["sm_mhz"], sampled["sm_max_mhz"], ", ".join(sampled["reasons"]) or "none"))
    for name, (times, nbytes) in (("(a) 8 kHz host clip 3 s", clip), ("(b) 8 kHz host live 240", live)):
        for k in times:
            print("%-24s %-6s %s ms per call (rounds); %.3f GB host-to-device per call" %
                  (name, k, " / ".join("%.2f" % t for t in times[k]), nbytes[k] / 1e9))
    for k in dev:
        print("%-24s %-6s %s ms per call (rounds)" % ("(c) 16 kHz device clip 3 s", k, " / ".join("%.2f" % t for t in dev[k])))


if __name__ == "__main__":
    main()
