"""The frontend kernels at the stream counts the benchmark runs, feature for feature (run with -m gpu on an H100).

frontend_clip_fuses (mww_frontend.cu) sends a call to the fused clip kernel k1_spectral_kernel<true, 4, T> -- three quarters
of the benchmark step -- only with more than 8 frames and at least 12 x SMs streams (1 584 on a 132-SM H100); below that the
unfused K1 + K2 pair runs.  So the tests here run tens of thousands of streams and compare every uint16 feature of every
stream, bit for bit, with the oracle frontend (and the final carry / noise estimate with oracle.Frontend.state()):

  1. the benchmark's shape (65 536 streams, two 48 000-sample calls: a partial last group of 10 frames, then a call entering
     with 320 carried samples and a carried estimate), for int16 and float32 audio;
  2. the same through an unaligned int16 view with call lengths that are not multiples of 8 (the per-sample loaders);
  3. the MWW_K1_OCC=3 instantiation k1_spectral_kernel<true, 3, T>, in a child process (the variable is read once per process);
  4. both sides of the switch point (12 x SMs - 1 and 12 x SMs streams) on one call sequence carrying state;
  5. live steps at scale (the fused short-call kernel, 5 streams per CTA, a partial last CTA);
  6. an int8 model engine whose calls are split into stream tiles (MWW_SCRATCH_MB): the fused kernel with non-zero offsets
     into carry and estimate, probabilities against the oracle and against an untiled engine.

Input layout as in test_gpu_full_size.py: P = 1021 distinct base streams, stream s carries base[s % P] (gathered on the
device); the oracle runs over the P base streams only.  Streams with the same content must also give bit-identical output.
The base streams are built to reach the frontend's edges: the edge-case rows, the host emulation's full-scale adversarial
families, an amplitude ladder that makes every input shift 0..15 occur, -32768 on the window's centre samples 238..241 (the
column k1_window_fft1 special-cases), noise-estimate stressors, and piecewise segment streams cut across frame, 16-frame-group
and call boundaries."""

import os
import subprocess
import sys

import numpy as np
import pytest

import oracle
from conftest import GOLDEN, ROOT, edge_case_audio, synth_audio
from test_gpu_full_size import check_streams, periodic_streams

pytestmark = pytest.mark.gpu

P = 1021
N = 96000                      # two benchmark calls of 48 000 samples
S_BENCH = 65536
S_LIVE = 65509                 # 13 101 CTAs of 5 streams + one of 4
HOP, WINDOW, CARRY = 160, 480, 320
ROWS = (N - WINDOW) // HOP + 1                                     # 598 = 298 + 300


# ---- base streams ----------------------------------------------------------------------------------------------------

def _piecewise(rng, n):
    """Segments of silence, DC, full-scale clipping, alternating extremes, tones, noise and impulses (the hypothesis test's
    kinds in test_host_emul.py), cut at random positions and next to frame starts, 16-frame-group starts and the call
    boundary (call 2's frames start 320 samples before its first sample: groups at 47 680 + 2 560 g)."""
    near = [48000, 47680 + 2560 * int(rng.integers(0, 19)), 2560 * int(rng.integers(1, 19)), 160 * int(rng.integers(3, 598))]
    cuts = {c + int(d) for c in near for d in rng.choice([-241, -240, -1, 0, 1, 79, 238, 241], 2)}
    cuts |= {int(c) for c in rng.integers(1, n, int(rng.integers(2, 12)))}
    cuts = sorted(c for c in cuts if 0 < c < n)
    x = np.zeros(n)
    for a, b in zip([0] + cuts, cuts + [n]):
        kind, amp, t = rng.integers(0, 7), int(rng.integers(0, 32768)), np.arange(b - a)
        if kind == 1:
            x[a:b] = amp if rng.random() < 0.5 else -amp - 1
        elif kind == 2:
            x[a:b] = rng.choice([-32768, 32767], b - a)
        elif kind == 3:
            x[a:b] = np.where(t % 2 == 0, amp, -amp - 1)
        elif kind == 4:
            x[a:b] = amp * np.sin(2 * np.pi * rng.uniform(50, 7950) / 16000.0 * t + rng.uniform(0, 6.3))
        elif kind == 5:
            x[a:b] = rng.normal(0, amp / 3 + 1, b - a)
        elif kind == 6:
            x[a + int(rng.integers(0, b - a))] = amp if rng.random() < 0.5 else -32768
    return x


def stress_audio(n=N, seed=2026):
    """[P, n] int16, pairwise distinct rows: the families of the module docstring, then synth_audio for the remainder."""
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    rows = list(edge_case_audio(n).astype(np.float64))
    for i in range(32):                      # test_host_emul.py's adversarial families, full length
        kind = i % 4
        if kind == 0:
            rows.append(rng.choice([-32768, 32767], n))
        elif kind == 1:
            rows.append(rng.integers(-32768, 32768, n))
        elif kind == 2:
            w = [np.pi / 2, np.pi / 4, np.pi / 8, 3 * np.pi / 8, np.pi / 16, 5 * np.pi / 8, 7 * np.pi / 8, rng.uniform(0, np.pi)][i // 4]
            rows.append(32767 * np.sign(np.cos(w * (t // 2) + rng.uniform(0, 6.28) + (t % 2) * np.pi / 2) + 1e-12))
        else:
            rows.append(rng.normal(0, 30000, n))
    peaks = sorted(({(1 << k) - 1 for k in range(16)} | {1 << k for k in range(16)}) - {0})
    for p in peaks:                          # every msb of the windowed maximum, so every input shift 0..15
        tone = np.clip(np.round(p * np.sin(2 * np.pi * rng.uniform(100, 7000) / 16000.0 * t)), -p, p)
        tone[::997] = -p
        noise = np.clip(np.round(rng.normal(0, p / 2.5 + 0.3, n)), -p, p)
        noise[::331] = p
        rows += [tone, noise]
    frames = np.arange(0, (n - WINDOW) // HOP + 1)
    for variant in range(4):                 # -32768 on window samples 238..241 of frames (the j == 7 column)
        x = [np.zeros(n), rng.normal(0, 100, n), np.where(rng.random(n) < 0.01, 32767, 0), rng.normal(0, 16384, n)][variant]
        if variant == 0:
            for j in range(238, 242):
                x[HOP * frames + j] = -32768
        else:
            x[HOP * frames + 238 + (frames + variant) % 4] = -32768
        rows.append(x)
    tone = 32767 * np.sin(2 * np.pi * 1000.0 * t / 16000.0)
    rows.append(np.where(t < 32000, tone, 0))                                  # 2 s full scale, then silence
    rows.append(np.where(t < 32000, tone, np.where(t % 2 == 0, 1, -1)))        # ... then +-1 dither
    rows.append(np.where((t // 32000) % 2 == 0, rng.normal(0, 20000, n), 0))   # noise and silence, 2 s each
    rows.append(rng.normal(0, 1000, n))                                        # stationary noise: signal ~ estimate
    rows.append(rng.normal(0, 30, n) + 500 * np.sin(2 * np.pi * 300.0 * t / 16000.0))
    rows.append(rng.choice([-1, 1], n))                                        # +-1 dither
    for _ in range(64):
        rows.append(_piecewise(rng, n))
    rows = [np.clip(np.round(r), -32768, 32767).astype(np.int16) for r in rows]
    rows += [synth_audio(n, seed + 1000 + i) for i in range(P - len(rows))]
    return np.stack(rows)


# ---- checks ----------------------------------------------------------------------------------------------------------

def check_features(torch, got, want, what, chunk=8192):
    """got uint16 CUDA [S, T, 40], want uint16 host [P, T, 40] (oracle over the base streams): streams with the same content
    are bit-identical, and stream s equals want[s % P].  A failure names the stream, frame and channel."""
    S, T, C = got.shape
    Pw = want.shape[0]
    assert want.shape == (Pw, T, C), (what, got.shape, want.shape)
    g_all = got.reshape(S, T * C).view(torch.int16)
    w_dev = torch.from_numpy(np.ascontiguousarray(want).reshape(Pw, T * C).view(np.int16)).to(got.device)
    first = g_all[:Pw]
    for s0 in range(0, S, chunk):
        g = g_all[s0:s0 + chunk]
        idx = torch.arange(s0, s0 + g.shape[0], device=got.device) % Pw
        for ref, kind in ((first.index_select(0, idx), "differs from stream s % P"), (w_dev.index_select(0, idx), "differs from the oracle")):
            bad = g != ref
            if bool(bad.any()):
                s, k = (int(v) for v in torch.nonzero(bad)[0])
                n_bad = int(bad.sum())
                raise AssertionError("%s: %s at stream %d (base %d), frame %d, channel %d: got %d, want %d (%d values in streams %d..%d)"
                                     % (what, kind, s0 + s, (s0 + s) % Pw, k // C, k % C, int(g[s, k]) & 0xFFFF, int(ref[s, k]) & 0xFFFF,
                                        n_bad, s0, s0 + g.shape[0] - 1))


def oracle_state(base):
    """(used, carry [P, 480], estimate [P, 40]) of oracle.Frontend after each whole base stream"""
    used, carry, est = None, np.zeros((base.shape[0], WINDOW), np.int16), np.zeros((base.shape[0], 40), np.uint32)
    for i, row in enumerate(base):
        fe = oracle.Frontend()
        fe.stream(row)
        buf, u, e = fe.state()
        assert used in (None, u)
        used, carry[i], est[i] = u, buf, e
    return used, carry, est


def check_state(st, want_state, what):
    used, carry, est = want_state
    S = st["carry"].shape[0]
    idx = np.arange(S) % carry.shape[0]
    assert st["frontend_buffered"] == used, (what, st["frontend_buffered"], used)
    bad = np.nonzero((st["carry"][:, :used] != carry[idx, :used]).any(1))[0]
    assert bad.size == 0, (what, "carry differs from the oracle's at streams", bad[:8].tolist())
    bad = np.nonzero((st["estimate"] != est[idx]).any(1))[0]
    assert bad.size == 0, (what, "noise estimate differs from the oracle's at streams", bad[:8].tolist())


class Inputs:
    """base [P, N] int16 (host), dev [S_BENCH, N] int16 (CUDA, stream s = base[s % P]), the oracle's features over the base
    streams and (lazily) its final frontend state"""

    def __init__(self, torch):
        self.torch = torch
        self.base = stress_audio()
        self.dev = periodic_streams(torch, self.base, S_BENCH, ())
        self.want, _ = oracle.run_pipeline(None, self.base, want_probs=False, threads=8)
        assert self.want.shape == (P, ROWS, 40)
        self._state = None

    def state(self):
        if self._state is None:
            self._state = oracle_state(self.base)
        return self._state

    def chunk(self, S, lo, hi, dtype="i16"):
        x = self.dev[:S, lo:hi].contiguous()
        return x.to(self.torch.float32).mul_(1.0 / 32768) if dtype == "f32" else x    # exact: to_int16 gives x back


@pytest.fixture(scope="module")
def inputs(torch_cuda):
    return Inputs(torch_cuda)


def features_call(eng, x, launches):
    l0 = eng.launch_count
    out = eng.features(x)
    assert eng.launch_count - l0 == launches, ("launches", eng.launch_count - l0, "expected", launches)
    return out


def run_bench_shape(inp, dtype, layout=None):
    """Case 1 (and 2 with layout = (storage offset, extra row pitch) and call lengths 47 999 + 48 001)."""
    from microwakeword_b200.engine import StreamEngine
    torch = inp.torch
    eng = StreamEngine(None, n_streams=S_BENCH)
    calls = (48000, 48000) if layout is None else (47999, 48001)
    pos, row = 0, 0
    for call, n in enumerate(calls):
        x = inp.chunk(S_BENCH, pos, pos + n, dtype)
        if layout is not None:
            x = unaligned(torch, x, *layout)
        buffered = eng.frontend_buffered
        out = features_call(eng, x, 2)                   # the fused clip kernel + the carry update
        T = (buffered + n - WINDOW) // HOP + 1
        assert out.shape == (S_BENCH, T, 40)
        if layout is None:
            assert (buffered, T % 16) == ((0, 10) if call == 0 else (CARRY, 300 % 16))
        check_features(torch, out, inp.want[:, row:row + T], (dtype, layout, "call", call))
        del out, x
        pos, row = pos + n, row + T
    assert (pos, row) == (N, ROWS)
    check_state(eng.state_dict(), inp.state(), (dtype, layout))


def unaligned(torch, x, offset, pitch_extra):
    """x [S, n] -> the same values in a tensor whose storage starts `offset` elements in and whose row pitch is n + pitch_extra
    (test_gpu_float_audio._unaligned, for int16)"""
    S, n = x.shape
    pitch = n + pitch_extra
    flat = torch.full((S * pitch + offset,), -12345, dtype=x.dtype, device=x.device)
    view = flat[offset:].view(S, pitch)[:, :n]
    view.copy_(x)
    assert view.storage_offset() == offset and view.stride() == (pitch, 1)
    return view


# ---- 1, 2, 3: the benchmark's shape ------------------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", ["i16", "f32"])
def test_fused_clip_kernel_at_benchmark_shape(inputs, dtype):
    run_bench_shape(inputs, dtype)


def test_fused_clip_kernel_per_sample_loaders(inputs):
    """storage offset 3 samples, row pitch n + 5, 47 999 then 48 001 samples: 297 rows leaving 479 carried samples, then 301"""
    run_bench_shape(inputs, "i16", layout=(3, 5))


def child_verdict():
    """Run case 1 (int16) in this process and return a one-line verdict, with the fused clip kernels the run launched."""
    import torch
    torch.cuda.init()
    inp = Inputs(torch)
    from torch.profiler import ProfilerActivity, profile
    from microwakeword_b200.engine import StreamEngine
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        StreamEngine(None, n_streams=S_BENCH).features(inp.chunk(S_BENCH, 0, 48000))
        torch.cuda.synchronize()
    names = sorted({e.key for e in prof.key_averages() if "k1_spectral_kernel" in e.key})
    try:
        run_bench_shape(inp, "i16")
    except AssertionError as e:
        return "FAIL %s | %s" % (names, str(e).replace("\n", " "))
    return "OK %s" % names


def test_occupancy_3_instantiation_at_benchmark_shape():
    """MWW_K1_OCC=3 selects k1_spectral_kernel<true, 3, T> (per-lane twiddles in registers); the frontend reads the variable
    once per process, so case 1 runs in a child process with a timeout."""
    env = dict(os.environ, MWW_K1_OCC="3")
    code = ("import sys; sys.path[:0] = [%r, %r]; import test_gpu_frontend_full_size as T; print('VERDICT', T.child_verdict())"
            % (ROOT, os.path.join(ROOT, "tests")))
    flags = ["-s"] if sys.flags.no_user_site else []
    res = subprocess.run([sys.executable] + flags + ["-c", code], env=env, cwd=ROOT, capture_output=True, text=True, timeout=1200)
    lines = [ln for ln in res.stdout.splitlines() if ln.startswith("VERDICT ")]
    assert res.returncode == 0 and len(lines) == 1, (res.returncode, res.stdout[-2000:], res.stderr[-4000:])
    verdict = lines[0][len("VERDICT "):]
    assert verdict.startswith("OK "), verdict
    assert "k1_spectral_kernel<true, 3," in verdict and "k1_spectral_kernel<true, 4," not in verdict, verdict


# ---- 4: the switch point -----------------------------------------------------------------------------------------------

SWITCH_CALLS = [(1760, 9), (2600, 16), (2700, 17), (5000, 31), (47700, 298)]     # (samples, frames); carried 320..400


@pytest.mark.parametrize("side", ["unfused", "fused"])
def test_switch_between_unfused_and_fused_clip_kernels(torch_cuda, inputs, side):
    """12 x SMs - 1 streams: unfused K1 (grid.y > 1 from 17 frames on) + K2 + carry update; 12 x SMs: the fused kernel +
    carry update.  The launch count pins the path; the features pin the arithmetic, carried state included."""
    from microwakeword_b200.engine import StreamEngine
    sms = torch_cuda.cuda.get_device_properties(0).multi_processor_count
    S = 12 * sms - (1 if side == "unfused" else 0)
    eng = StreamEngine(None, n_streams=S)
    pos, row = 0, 0
    for n, frames in SWITCH_CALLS:
        out = features_call(eng, inputs.chunk(S, pos, pos + n), 3 if side == "unfused" else 2)
        assert out.shape == (S, frames, 40)
        check_features(torch_cuda, out, inputs.want[:, row:row + frames], (side, S, n))
        pos, row = pos + n, row + frames


# ---- 5: live steps at scale --------------------------------------------------------------------------------------------

def test_live_steps_at_scale(torch_cuda, inputs):
    """one 1 760-sample call (9 frames: fused clip kernel), then 48 calls of 480 samples (3 frames: k1k2_packed_kernel, one
    launch, 5 streams per CTA, the last CTA partial)"""
    from microwakeword_b200.engine import StreamEngine
    S = S_LIVE
    assert S % 5 != 0
    eng = StreamEngine(None, n_streams=S)
    got = [features_call(eng, inputs.chunk(S, 0, 1760), 2)]
    pos = 1760
    for _ in range(48):
        got.append(features_call(eng, inputs.chunk(S, pos, pos + 480), 1))
        assert got[-1].shape == (S, 3, 40)
        pos += 480
    got = torch_cuda.cat(got, 1)
    check_features(torch_cuda, got, inputs.want[:, :got.shape[1]], "live")


# ---- 6: stream tiles ---------------------------------------------------------------------------------------------------

def test_tiled_int8_clip_calls(torch_cuda, inputs, monkeypatch):
    """MWW_SCRATCH_MB=256: the 3 s calls split into 6 tiles of <= 11 259 streams (the last partial), so the fused kernel runs
    with non-zero offsets into carry and estimate.  Probabilities bit-exact against the oracle and an untiled engine; the
    final states identical."""
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    with open(os.path.join(GOLDEN, "okay_nabu_synth_int8.mww"), "rb") as f:
        blob = f.read()
    plain = StreamEngine(blob, n_streams=S_BENCH)
    monkeypatch.setenv("MWW_SCRATCH_MB", "256")                   # read at mww_create
    tiled = StreamEngine(blob, n_streams=S_BENCH)
    for frames in (298, 300):
        tile = (256 << 20) // (frames * 40 * 2)                    # mww_capi.cu tile_streams: feature scratch only (fused)
        assert -(-S_BENCH // tile) >= 5 and S_BENCH % tile != 0
    got, pos = [], 0
    for n in (48000, 48000):
        x = inputs.chunk(S_BENCH, pos, pos + n)
        l0 = tiled.launch_count
        a = tiled.predict_clip(x)
        assert tiled.launch_count - l0 >= 2 * 5 + 1, "the call was not tiled"
        b = plain.predict_clip(x)
        assert torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32)), ("tiled != untiled", n)
        got.append(a)
        pos += n
    _, want = oracle.run_pipeline(blob, inputs.base, want_features=False, threads=8)
    got = torch.cat(got, 1)
    assert got.shape == (S_BENCH, 199) and want.shape == (P, 199)
    check_streams(torch, got, want, True, "tiled int8")
    st_t, st_p = tiled.state_dict(), plain.state_dict()
    for k in st_p:
        assert np.array_equal(np.asarray(st_t[k]), np.asarray(st_p[k])), k
    check_state(st_t, inputs.state(), "tiled")
