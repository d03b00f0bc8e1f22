"""What a sample format per stream costs: 65 536 streams of an fp32 okay_nabu engine with per-stream rates, a quarter each of
8 kHz mu-law, 8 kHz A-law, 48 kHz float32 and 16 kHz int16 (in that order, each quarter a block of neighbouring slots).
Three arms on the same rates, alternated round by round, outputs compared bit for bit:
  mixed      one step(mixed=True) on the uint8 rows (mww_predict_clip_mixed);
  int16      (a) one step on rows holding the same samples as int16 (already decoded, outside the timing);
  torch+s16  (b) the mixed rows decoded in torch into an int16 buffer, then one int16 step.
30 ms live calls from device memory, ms per call from CUDA events, the best of --rounds rounds of --calls calls; and one 3 s
call through predict_clip_host from pinned memory at --host-streams streams (MWW_MIN_TILE_STREAMS=128, so that the staged
tiles follow the blocks), mixed against int16, ms from the host clock, with the bytes each copies.  Prints the card, its
power limit and the SM clock.  There is no CPU path: without a GPU it fails.
    python tools/stream_formats_time.py [--streams 65536] [--host-streams 2048] [--rounds 5] [--calls 50]"""
import argparse
import os
import sys
import time

os.environ.setdefault("MWW_MIN_TILE_STREAMS", "128")
import numpy as np  # noqa: E402
import torch  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench import ClockSampler, model_blob  # noqa: E402
from event_positions_time import card, event_time  # noqa: E402
from microwakeword_b200.engine import SAMPLE_FORMATS, StreamEngine, bytes_for_formats, inputs_for_rates  # noqa: E402

MIX = ((8000, "ulaw"), (8000, "alaw"), (48000, "f32"), (16000, "s16"))


def ulaw_table():
    u = (~np.arange(256)) & 0xFF
    t = (((u & 0x0F) << 3) + 0x84) << ((u & 0x70) >> 4)
    return np.where(u & 0x80, 0x84 - t, t - 0x84).astype(np.int16)


def alaw_table():
    a = np.arange(256) ^ 0x55
    t, seg = (a & 0x0F) << 4, (a & 0x70) >> 4
    t = np.where(seg == 0, t + 8, np.where(seg == 1, t + 0x108, (t + 0x108) << np.maximum(seg - 1, 0)))
    return np.where(a & 0x80, t, -t).astype(np.int16)


def layout(S):
    q = S // 4
    rates = np.repeat([r for r, _ in MIX], q).astype(np.int32)
    fmts = np.repeat([SAMPLE_FORMATS[f] for _, f in MIX], q).astype(np.int32)
    return rates, fmts, q


def rows(rng, rates, fmts, q, t, n16):
    """(mixed uint8 rows, the same samples as int16 rows), numpy"""
    S = rates.size
    D = inputs_for_rates(rates, t, n16)
    width = int(bytes_for_formats(rates, fmts, t, n16).max() + 3) // 4 * 4
    x = np.zeros((S, width), np.uint8)
    y = np.zeros((S, int(D.max())), np.int16)
    lut = {"ulaw": ulaw_table(), "alaw": alaw_table()}
    for b, (r, f) in enumerate(MIX):
        blk, d = slice(b * q, (b + 1) * q), int(D[b * q])
        if f in lut:
            c = rng.integers(0, 256, (q, d)).astype(np.uint8)
            x[blk, :d], y[blk, :d] = c, lut[f][c]
        elif f == "f32":
            v = (rng.standard_normal((q, d)) * 0.3).astype(np.float32)
            x[blk, :4 * d] = v.view(np.uint8)
            y[blk, :d] = np.clip(v * 32768, -32768, 32767).astype(np.int16)
        else:
            v = (rng.standard_normal((q, d)) * 9000).clip(-32768, 32767).astype(np.int16)
            x[blk, :2 * d], y[blk, :d] = v.view(np.uint8), v
    return x, y


class TorchDecode:
    """arm (b): the mixed rows decoded in torch into one int16 buffer"""

    def __init__(self, q, D, width16, dev):
        self.q, self.D = q, D
        self.lut = {f: torch.from_numpy(t).to(dev) for f, t in (("ulaw", ulaw_table()), ("alaw", alaw_table()))}
        self.out = torch.zeros((4 * q, width16), dtype=torch.int16, device=dev)

    def __call__(self, x):
        q = self.q
        for b, (_, f) in enumerate(MIX):
            d, blk, o = int(self.D[b * q]), x[b * q:(b + 1) * q], self.out[b * q:(b + 1) * q]
            if f in self.lut:
                o[:, :d] = self.lut[f][blk[:, :d].long()]
            elif f == "f32":
                o[:, :d] = (blk[:, :4 * d].contiguous().view(torch.float32) * 32768).clamp(-32768, 32767).to(torch.int16)
            else:
                o[:, :d] = blk[:, :2 * d].contiguous().view(torch.int16)
        return self.out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--streams", type=int, default=65536)
    ap.add_argument("--host-streams", type=int, default=2048)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("stream_formats_time.py needs a CUDA device (there is no CPU path)")
    print("card: %s" % card())
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(1)
    blob = model_blob("f32")
    clocks = ClockSampler(0)
    try:
        run(a, dev, rng, blob)
    finally:
        print("SM clock during the run: %s" % clocks.stop())


def run(a, dev, rng, blob):
    # ---- 30 ms live calls, device-resident rows: the calls of a round reuse one call's rows (t advances by 480 each time, and
    # every 30 ms call at these rates holds the same number of samples)
    rates, fmts, q = layout(a.streams)
    x, y = rows(rng, rates, fmts, q, 0, 480)
    dx, dy = torch.from_numpy(x).to(dev), torch.from_numpy(y).to(dev)
    mixed = StreamEngine(blob, a.streams, 0, stream_rates=rates, stream_formats=fmts)
    s16 = StreamEngine(blob, a.streams, 0, stream_rates=rates)
    tdec = StreamEngine(blob, a.streams, 0, stream_rates=rates)
    dec = TorchDecode(q, inputs_for_rates(rates, 0, 480), y.shape[1], dev)
    arms = {"mixed": lambda: mixed.step(dx, mixed=True), "int16": lambda: s16.step(dy), "torch+s16": lambda: tdec.step(dec(dx))}
    outs = {k: f() for k, f in arms.items()}
    assert torch.equal(outs["mixed"], outs["int16"]) and torch.equal(outs["mixed"], outs["torch+s16"]), "arms differ"
    best = {k: [] for k in arms}
    for _ in range(a.rounds):
        for k, f in arms.items():
            best[k].append(event_time(f, a.calls))
        outs = {k: f() for k, f in arms.items()}
        assert torch.equal(outs["mixed"], outs["int16"]) and torch.equal(outs["mixed"], outs["torch+s16"]), "arms differ"
    print("live 30 ms, %d streams (bytes per call: mixed %d, int16 %d)" % (a.streams, x.nbytes, y.nbytes))
    for k in arms:
        print("  %-10s %.4f ms per call (rounds: %s)" % (k, min(best[k]), " ".join("%.4f" % v for v in best[k])))
    del mixed, s16, tdec, dec, dx, dy
    torch.cuda.empty_cache()

    # ---- one 3 s call through predict_clip_host, pinned rows
    rates, fmts, q = layout(a.host_streams)
    mixed = StreamEngine(blob, a.host_streams, 0, stream_rates=rates, stream_formats=fmts)
    s16 = StreamEngine(blob, a.host_streams, 0, stream_rates=rates)
    x, y = rows(rng, rates, fmts, q, 0, 48000)
    hx, hy = mixed.host_buffer(x.shape, np.uint8), s16.host_buffer(y.shape, np.int16)
    hx[:], hy[:] = x, y
    D = inputs_for_rates(rates, 0, 48000)
    moved = sum(int(bytes_for_formats(rates[b * q:(b + 1) * q], fmts[b * q:(b + 1) * q], 0, 48000).max() + 3) // 4 * 4 * q for b in range(4))
    times = {"mixed": [], "int16": []}
    for r in range(a.rounds):
        for k, e, buf in (("mixed", mixed, hx), ("int16", s16, hy)):
            e.reset()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = e.predict_clip_host(buf, samples16=48000, mixed=k == "mixed")
            times[k].append((time.perf_counter() - t0) * 1e3)
            if k == "mixed":
                want = out.copy()
            else:
                assert np.array_equal(out, want), "host arms differ"
    print("3 s predict_clip_host, %d streams, %d tiles of 128 (bytes copied: mixed %d in tiles as wide as their widest row, "
          "int16 %d)" % (a.host_streams, a.host_streams // 128, moved, int(D.max()) * 2 * a.host_streams))
    for k in times:
        print("  %-10s %.2f ms per call (rounds: %s)" % (k, min(times[k]), " ".join("%.2f" % v for v in times[k])))


if __name__ == "__main__":
    main()
