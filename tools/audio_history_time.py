"""What the audio history costs: the same calls on two fp32 okay_nabu engines at --streams (65 536 by default), one without a
history and one with set_audio_history(--capacity, 32 000 = 2 s by default), alternating inside each round; the best round
of each arm is the figure.  Their probabilities must be bit-identical (checked).

  (a) live ........ 480-sample step() calls on device-resident int16 audio (the fused short-call kernel, then one append)
  (b) device clip . 3 s predict_clip calls (48 000 samples) on device-resident int16 audio (the call is longer than the ring:
                    only its last capacity samples are written)
  (c) host ulaw ... an 8 kHz handle's 3 s predict_clip_host calls (24 000 mu-law codes per stream) from pinned host memory:
                    resampled, then appended from the 16 kHz tile scratch, tile by tile
  (d) read ........ audio_history of --read-ids streams x 24 000 samples (1.5 s) into a preallocated tensor, by a device id
                    list and by a host id list, after a call that leaves the ring's read start unaligned and after one that
                    leaves it aligned
Times in ms per call: CUDA events around device calls, the host wall clock around the synchronous host calls.  Prints the
card, its power limit and the SM clock sampled during the run.  There is no CPU path: without a GPU it fails.
    python tools/audio_history_time.py [--streams 65536] [--capacity 32000] [--rounds 5] [--read-ids 1024]"""
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


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "%s (nvidia-smi unavailable)" % torch.cuda.get_device_name(0)


def device_audio(S, n, seed):
    idx = torch.arange(S, device="cuda") % P
    return synth_audio_device(torch, P, n, seed, torch.device("cuda", 0))[idx].contiguous()


def engines(S, capacity, rate=16000):
    blob = model_blob("f32")
    eng = {"off": StreamEngine(blob, n_streams=S, input_rate=rate), "on": StreamEngine(blob, n_streams=S, input_rate=rate)}
    eng["on"].set_audio_history(capacity)
    return eng


def event_time(fn, calls):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(calls):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / calls


def device_arms(S, capacity, n, calls, rounds):
    """(a) / (b): -> {arm: [ms per call per round]}"""
    audio = device_audio(S, n, 3)
    eng = engines(S, capacity)
    out = {k: torch.empty((S, 128), dtype=torch.float32, device="cuda") for k in eng}
    last = {}
    fn = {k: (lambda k=k: last.__setitem__(k, eng[k].predict_clip(audio, out=out[k]))) for k in eng}
    for k in eng:
        for _ in range(3):
            fn[k]()
    times = {k: [] for k in eng}
    for _ in range(rounds):
        for k in eng:
            times[k].append(event_time(fn[k], calls))
    assert torch.equal(last["off"].view(torch.int32), last["on"].view(torch.int32))
    assert eng["on"].audio_samples_seen > 0
    for e in eng.values():
        e.close()
    return times


def ulaw_codes(S, n):
    """uint8 [S, n] mu-law codes of the benchmark's synthetic audio, pinned"""
    u = (~np.arange(256)) & 0xFF
    t = (((u & 0x0F) << 3) + 0x84) << ((u & 0x70) >> 4)
    table = np.where(u & 0x80, 0x84 - t, t - 0x84).astype(np.int16)
    order = np.argsort(table, kind="stable")
    x = synth_audio_device(torch, P, n, 5, torch.device("cuda", 0)).cpu().numpy()
    base = order[np.minimum(np.searchsorted(table[order], x), 255)].astype(np.uint8)
    out = host_array((S, n), np.uint8)
    for s0 in range(0, S, P):
        out[s0:s0 + P] = base[:min(P, S - s0)]
    return out


def host_arms(S, capacity, calls, rounds):
    """(c): -> {arm: [ms per call per round]}"""
    codes = ulaw_codes(S, 24000)
    eng = engines(S, capacity, rate=8000)
    out = {k: host_array((S, 128), np.float32) for k in eng}
    last = {}
    for k in eng:
        for _ in range(2):
            last[k] = eng[k].predict_clip_host(codes, out=out[k], law="ulaw")
    times = {k: [] for k in eng}
    for _ in range(rounds):
        for k in eng:
            t0 = time.perf_counter()
            for _ in range(calls):
                last[k] = eng[k].predict_clip_host(codes, out=out[k], law="ulaw")
            times[k].append((time.perf_counter() - t0) * 1e3 / calls)
    assert np.array_equal(last["off"].view(np.int32), last["on"].view(np.int32))
    for e in eng.values():
        e.close()
    return times


def read_arms(S, capacity, n_ids, n_samples, calls, rounds):
    """(d): -> {form: [ms per read per round]}, bytes a read moves"""
    eng = StreamEngine(None, n_streams=S)
    eng.set_audio_history(capacity)
    audio = device_audio(S, 48000, 11)
    eng.features(audio)
    ids = torch.randperm(S, device="cuda")[:n_ids].to(torch.int32)
    host_ids = ids.cpu().numpy()
    out = torch.empty((n_ids, n_samples), dtype=torch.int16, device="cuda")
    times = {}
    for start, extra in (("unaligned start", 4), ("aligned start", 4)):
        eng.features(audio[:, :extra])             # 4, then 8 samples past a multiple of 8: the read start moves with it
        for form, fn in (("device ids", lambda: eng.audio_history(ids, n_samples, out=out)),
                         ("host ids", lambda: eng.audio_history(host_ids, n_samples, out=out))):
            fn()
            times["%s, %s" % (form, start)] = [event_time(fn, calls) for _ in range(rounds)]
    want = audio[ids.long(), 48000 - n_samples + 8:]
    tail = audio[ids.long(), :4]
    assert torch.equal(out[:, :n_samples - 8], want) and torch.equal(out[:, n_samples - 8:], torch.cat([tail, tail], 1))
    eng.close()
    return times, 2 * n_ids * n_samples * 2


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--streams", type=int, default=65536)
    ap.add_argument("--capacity", type=int, default=32000)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--live-calls", type=int, default=50)
    ap.add_argument("--clip-calls", type=int, default=3)
    ap.add_argument("--read-ids", type=int, default=1024)
    ap.add_argument("--read-samples", type=int, default=24000)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("audio_history_time.py measures the GPU kernels and needs a CUDA device; none is available")
    S = a.streams
    print("card: %s; %d streams, fp32 okay_nabu, history capacity %d samples" % (card(), S, a.capacity))
    clocks = ClockSampler(0)
    try:
        live = device_arms(S, a.capacity, 480, a.live_calls, a.rounds)
        torch.cuda.empty_cache()
        clip = device_arms(S, a.capacity, 48000, a.clip_calls, a.rounds)
        torch.cuda.empty_cache()
        host = host_arms(S, a.capacity, a.clip_calls, a.rounds)
        torch.cuda.empty_cache()
        reads, nbytes = read_arms(S, a.capacity, a.read_ids, a.read_samples, 20, a.rounds)
    finally:
        sampled = clocks.stop()
    print("SM clock during the run: median %s MHz (max %s MHz), throttle reasons seen: %s" %
          (sampled["sm_mhz"], sampled["sm_max_mhz"], ", ".join(sampled["reasons"]) or "none"))
    for name, times in (("(a) live 480", live), ("(b) device clip 3 s", clip), ("(c) 8 kHz ulaw host clip 3 s", host)):
        for k in times:
            print("%-30s history %-4s best %.3f ms per call (rounds %s)" % (name, k, min(times[k]), " / ".join("%.3f" % t for t in times[k])))
    for k, t in reads.items():
        print("%-30s %-28s best %.4f ms per read (%.1f GB/s of %d bytes read + written)" %
              ("(d) read %d x %d" % (a.read_ids, a.read_samples), k, min(t), nbytes / min(t) / 1e6, nbytes))


if __name__ == "__main__":
    main()
