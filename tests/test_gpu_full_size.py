"""The NN kernels at the stream counts the benchmark runs (run with -m gpu on an H100).

Most NN kernels are persistent: a CTA walks work items (one stream for the wgmma clip kernel, a group of 32 streams for the
live-step kernels) with a grid stride, so the code a CTA runs for its second and later items -- barrier hand-offs guarded by
the iteration count, mbarrier phases carried across groups, a window loaded one period early, buffers reloaded per stream --
only runs once the streams outnumber the grid.  Every test here gives each kernel it targets at least three waves.

Input layout: P distinct base streams, P prime; stream s carries base[s % P] (gathered on the device) and the CPU oracle runs over
the P base streams only.  The stream the same CTA handled one item earlier is s - grid (clip kernel) or s - 32 grid (live
kernels); a prime P that divides neither step (asserted for grids of 1, 2 and 4 x SMs) gives the two streams different content,
so a stale buffer or a read of the wrong group cannot reproduce the right answer by coincidence.

Two checks on every output: (i) stream s matches oracle[s % P] -- bit-exact for int8, within F32_TOL for fp32; (ii) all streams
with the same content give bit-identical outputs.  (ii) does not lean on the oracle's tolerance: every kernel computes a stream
with the same instructions in the same order whatever its slot (the MMA rows of a group are independent, the depthwise taps are
summed in ring order, which all streams of a handle share)."""

import os

import numpy as np
import pytest

import oracle
from conftest import GOLDEN, edge_case_audio, synth_audio
from oracle import detection_ref as D

pytestmark = pytest.mark.gpu

F32_TOL = 1e-5
STATE_TOL = 1e-4               # fp32 ring state after live steps vs after clip calls (summation order differs)
FEATURE_SCALE = np.float32(0.0390625)
P_AUDIO, P_ROWS = 1021, 257


def _blob(name):
    with open(os.path.join(GOLDEN, name), "rb") as f:
        return f.read()


def _is_prime(n):
    return n > 1 and all(n % d for d in range(2, int(n ** 0.5) + 1))


def _persistent_grids(sms, S):
    """{kernel: (grid, work items)} of the persistent NN kernels at S streams, sized as their launchers size them."""
    groups = -(-S // 32)
    return {"clip_tc": (min(S, 2 * sms), S),            # mww_nn_tc.cu: one stream per item, two CTAs per SM
            "live_v1": (min(groups, 2 * sms), groups),  # mww_nn_live.cu: groups of 32 streams
            "live_v2": (min(groups, sms), groups),
            "live_v3": (min(groups, sms), groups),
            "live_i8": (min(groups, 4 * sms), groups)}  # mww_nn_i8_live.cu


def periodic_streams(torch, base, S, kernels):
    """base [P, ...] (host) -> CUDA tensor [S, ...] with stream s = base[s % P].  Asserts that the period separates every stream
    from the one its CTA handled an item earlier, and that S gives each of `kernels` (keys of _persistent_grids) >= 3 waves."""
    P = base.shape[0]
    assert _is_prime(P), P
    assert len({row.tobytes() for row in base}) == P, "base streams must be pairwise distinct"
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for grid in (sms, 2 * sms, 4 * sms):
        for step in (grid, 32 * grid):       # P prime: step % P != 0 also keeps s - k step apart for every k < P
            assert step % P != 0, (grid, step, P)
    grids = _persistent_grids(sms, S)
    for k in kernels:
        grid, items = grids[k]
        assert items >= 3 * grid, (k, grid, items)
    u16 = base.dtype == np.uint16
    src = torch.from_numpy(np.ascontiguousarray(base.view(np.int16) if u16 else base)).cuda()
    out = src.index_select(0, torch.arange(S, device="cuda") % P)
    return out.view(torch.uint16) if u16 else out


def check_streams(torch, got, want, exact, what=""):
    """got [S, T] CUDA float32, want [P, >= T] oracle over the base streams: (ii) then (i) of the module docstring."""
    S, T = got.shape
    P = want.shape[0]
    idx = torch.arange(S, device=got.device) % P
    bits = got.contiguous().view(torch.int32)
    same = (bits == bits.index_select(0, idx)).all(1)
    assert bool(same.all()), ("streams with the same content differ", what, torch.nonzero(~same)[:8, 0].tolist())
    w = torch.from_numpy(np.ascontiguousarray(want[:, :T], np.float32)).to(got.device).index_select(0, idx)
    if exact:
        assert torch.equal(got, w), what
    else:
        err = (got - w).abs().max().item()
        assert err <= F32_TOL, (what, err)


def _f32_rows(torch, rows):
    """uint16 feature rows (CUDA) -> the float32 rows the reference feeds its model (u x 0.0390625: exact in float32)."""
    return (rows.view(torch.int16).to(torch.int32) & 0xFFFF).to(torch.float32) * float(FEATURE_SCALE)


def _base_audio(P, n, seed):
    """P distinct streams: the 14 edge cases, the rest seeded synthetic audio."""
    edge = edge_case_audio(n)
    return np.concatenate([np.stack([synth_audio(n, seed + i) for i in range(P - edge.shape[0])]), edge])


# ---- a. fp32 clip at the benchmark's shape -----------------------------------------------------------------------------

@pytest.fixture(scope="module")
def bench_clip(torch_cuda):
    """bench.py's flagship step: 65 536 streams, predict_clip on one 3 s buffer, twice.  Returns the two calls' probabilities
    (host, [S, 99] and [S, 100]) and the oracle over the base streams' buffer concatenated with itself."""
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    S, N = 65536, 48000
    blob = _blob("okay_nabu_synth_f32.mww")
    base = _base_audio(P_AUDIO, N, 7000)
    dev = periodic_streams(torch, base, S, ("clip_tc",))
    eng = StreamEngine(blob, n_streams=S)
    outs = []
    for call in range(2):
        # first call: 298 rows -> 99 steps, 1 row pending; second: 320 buffered samples + 48 000 -> 300 rows -> 100 steps.
        # Both >= 16 steps of uint16 rows: the wgmma kernel
        assert (eng.pending_rows, eng.frontend_buffered) == ((0, 0) if call == 0 else (1, 320))
        buf = torch.empty((S, 100), dtype=torch.float32, device="cuda")
        outs.append(eng.predict_clip(dev, out=buf).clone())
    del eng, dev
    _, want = oracle.run_pipeline(blob, np.concatenate([base, base], 1), want_features=False, threads=8)
    return outs, want


def test_fp32_clip_at_benchmark_shape(torch_cuda, bench_clip):
    (first, second), want = bench_clip
    assert first.shape == (65536, 99) and second.shape == (65536, 100) and want.shape == (P_AUDIO, 199)
    check_streams(torch_cuda, first, want[:, :99], False, "first call")
    check_streams(torch_cuda, second, want[:, 99:], False, "second call")


# ---- b. wgmma chunk boundaries across waves ----------------------------------------------------------------------------

# (row dtype, rows): steps = (pending + rows) // 3.  uint16 calls of >= 16 steps take the wgmma kernel, entering with 0, 1 and 2
# pending rows and ending on both sides of its 128-step chunks; the float32 call and the 8-step call take the mma.sync kernel
INFER_CALLS = [("u16", 48),     # p 0 -> 16 steps, p 0
               ("u16", 193),    # p 0 -> 64, p 1
               ("u16", 196),    # p 1 -> 65, p 2
               ("u16", 379),    # p 2 -> 127, p 0
               ("f32", 61),     # p 0 -> 20, p 1   (mma.sync: float32 rows)
               ("u16", 383),    # p 1 -> 128, p 0
               ("u16", 26),     # p 0 -> 8, p 2    (mma.sync: < 16 steps)
               ("u16", 385),    # p 2 -> 129, p 0
               ("u16", 772)]    # p 0 -> 257, p 1


def test_wgmma_chunk_boundaries_across_waves(torch_cuda):
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    S = 6 * sms + 37                             # every CTA of the 2-per-SM grid gets >= 3 streams; the last wave is partial
    total = sum(r for _, r in INFER_CALLS)
    blob = _blob("okay_nabu_synth_f32.mww")
    audio = _base_audio(P_ROWS, 480 + 160 * (total - 1), 7500)
    # features and, over exactly those rows, oracle.MixedNet.predict_u16 per base stream (run_pipeline does both, threaded)
    feats, want = oracle.run_pipeline(blob, audio, threads=8)
    assert feats.shape == (P_ROWS, total, 40) and want.shape == (P_ROWS, total // 3)
    rows = periodic_streams(torch, feats, S, ("clip_tc",))
    eng = StreamEngine(blob, n_streams=S)
    got, pos, pend = [], 0, 0
    for kind, r in INFER_CALLS:
        assert eng.pending_rows == pend
        chunk = rows.view(torch.int16)[:, pos:pos + r].contiguous().view(torch.uint16)
        if kind == "f32":
            chunk = _f32_rows(torch, chunk)
        out = eng.infer(chunk)
        assert out.shape == (S, (pend + r) // 3), (kind, r)
        got.append(out)
        pos, pend = pos + r, (pend + r) % 3
    assert [g.shape[1] for g in got] == [16, 64, 65, 127, 20, 128, 8, 129, 257]
    check_streams(torch, torch.cat(got, 1), want, False, "infer sequence")


# ---- c. live steps at scale --------------------------------------------------------------------------------------------

S_LIVE = 65509                 # 2^16 - 27: the short last group (5 streams) falls in a late wave of every live grid
LIVE_N = 31200                 # the longest sequence below: 2080 + 48 x 480 + 2000 + 8 x 480 = 30 960 samples


@pytest.fixture(scope="module")
def live_audio(torch_cuda):
    base = _base_audio(P_AUDIO, LIVE_N, 8000)
    dev = periodic_streams(torch_cuda, base, S_LIVE, ("clip_tc", "live_v1", "live_v2", "live_v3", "live_i8"))
    cache = {}

    def want(kind):
        if kind not in cache:
            cache[kind] = oracle.run_pipeline(_blob("okay_nabu_synth_%s.mww" % kind), base, want_features=False, threads=8)[1]
        return cache[kind]
    return dev, want


# (model and live kernel, pending rows entering every live step, how rows reach the NN).  "f32_rows": a frontend-only engine
# makes the rows and the live steps get them as float32 [S, 3, 40] through infer()
LIVE_CASES = [(k, p, "audio") for k in ("f32_v3", "f32_v2", "f32_v1", "int8") for p in (0, 1, 2)] + \
             [("f32_v3", 2, "f32_rows"), ("f32_v2", 1, "f32_rows"), ("f32_v1", 0, "f32_rows")]


@pytest.mark.parametrize("kind,pend,feed", LIVE_CASES)
def test_live_steps_at_scale(torch_cuda, live_audio, kind, pend, feed, monkeypatch):
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    dev, want = live_audio
    S = S_LIVE
    model = "int8" if kind == "int8" else "f32"
    if kind != "int8":
        monkeypatch.setenv("MWW_LIVE_VARIANT", kind[-1])        # read at mww_create
    blob = _blob("okay_nabu_synth_%s.mww" % model)
    exact = model == "int8"
    eng = StreamEngine(blob, n_streams=S)
    fe = StreamEngine(None, n_streams=S) if feed == "f32_rows" else None

    def call(n, live):
        chunk = dev[:, pos:pos + n].contiguous()
        if fe is None:
            return eng.predict_clip(chunk)
        rows = fe.features(chunk)
        if live:
            rows = _f32_rows(torch, rows)
            assert rows.shape == (S, 3, 40)
        return eng.infer(rows)

    got, pos = [], 0
    n0 = 1760 + 160 * pend                       # 9 + pend rows: 3 steps, `pend` rows left pending
    got.append(call(n0, False))
    pos += n0
    assert eng.pending_rows == pend
    for n_live in (48, 8):                       # 48 steps: every ring (4..22 rows) wraps at least twice
        for _ in range(n_live):
            got.append(call(480, True))
            pos += 480
            assert got[-1].shape == (S, 1)
        if n_live == 48:
            got.append(call(2000, False))        # a clip call: the rings are rotated back at full size
            pos += 2000
    assert eng.pending_rows == pend
    got = torch.cat(got, 1)
    assert got.shape == (S, 63)
    check_streams(torch, got, want(model), exact, (kind, pend, feed))
    del got
    # the state equals that of an engine that ran only clip calls over the same samples
    clip = StreamEngine(blob, n_streams=S)
    clip.predict_clip(dev[:, :pos].contiguous())
    a, b = eng.state_dict(), clip.state_dict()
    del eng, clip
    carry = fe.state_dict()["carry"] if fe is not None else a["carry"]
    assert np.array_equal(carry, b["carry"]) and np.array_equal(a["pending"], b["pending"])
    assert a["pending_rows"] == b["pending_rows"] == pend
    assert np.array_equal(a["nn"], b["nn"]) if exact else np.abs(a["nn"] - b["nn"]).max() <= STATE_TOL


# ---- d. int8 clip at full size -----------------------------------------------------------------------------------------

def test_full_size_properties(torch_cuda):
    """BASELINE.json configs[1] scale (65 536 streams) through the int8 clip kernel, which launches one CTA per stream: every
    stream against the oracle, replicas bit-identical, and chunked streaming at full size equal to the whole-clip call."""
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    S, N = 65536, 4800
    base = _base_audio(P_AUDIO, N, 600)
    dev = periodic_streams(torch, base, S, ())
    blob = _blob("okay_nabu_synth_int8.mww")
    eng = StreamEngine(blob, n_streams=S)
    got = eng.predict_clip(dev)
    assert got.shape == (S, 9)
    _, want = oracle.run_pipeline(blob, base, want_features=False, threads=8)
    check_streams(torch, got, want, True, "whole")
    eng.reset()
    a = eng.predict_clip(dev[:, :1760].contiguous())
    b = eng.predict_clip(dev[:, 1760:].contiguous())
    assert torch.equal(torch.cat([a, b], 1), got)


# ---- e. detection over 65 536 tracks -----------------------------------------------------------------------------------

def test_detection_over_full_size_tracks(torch_cuda, bench_clip):
    """moving_average / false_accept_counts / positive_scores over the 65 536 probability tracks of the benchmark step.  Tracks
    with the same content are bit-identical (test a), so the oracle runs over the P base tracks."""
    from microwakeword_b200 import detection as G
    (first, second), _ = bench_clip
    probs = torch_cuda.cat([first, second], 1).cpu().numpy()
    S, P = probs.shape[0], P_AUDIO
    idx = np.arange(S) % P
    assert np.array_equal(probs.view(np.int32), probs[idx].view(np.int32))
    tracks = list(probs)
    cutoffs = np.arange(0, 1.01, 0.01)
    moving = G.moving_average(tracks, 5)
    assert len(moving) == S
    want_ma = np.stack([D.moving_average(t, 5) for t in tracks[:P]])
    assert np.array_equal(np.stack(moving), want_ma[idx])
    counts = G.false_accept_counts(tracks, cutoffs, 25, window=5)
    want_fa = np.stack([D.false_accept_counts(m, cutoffs, 25) for m in want_ma])
    assert counts.shape == (S, cutoffs.size) and np.array_equal(counts, want_fa[idx])
    scores = G.positive_scores(tracks, 5, 25)
    want_ps = np.asarray([D.positive_score(t, 5, 25) for t in tracks[:P]], np.float32)
    assert np.array_equal(scores, want_ps[idx])
