"""The fused clip frontend k1_clip_kernel (half-warp phase boundaries, one CTA per stream) beyond the benchmark's shape, which
test_gpu_frontend_full_size.py covers (run with -m gpu on an H100).

Four CTAs fit an SM, so one wave is 4 x SMs CTAs (528 on a 132-SM H100).  The checks here run 12 x SMs streams (three waves
exactly, the smallest count the fused path takes), one stream more (a last wave of one CTA) and 65 509 streams; stream tiles
(MWW_SCRATCH_MB) whose last tile is 4 x SMs - 1 streams, less than one wave; two consecutive calls each, so the noise estimate
and the window carry continue across calls; and float32 and mu-law clips, each beside an int16 twin fed the same samples.
Features, carry and estimate must be bit-identical to the oracle frontend's and to the twin's.

Input layout as in test_gpu_frontend_full_size.py: stream s carries base[s % P] of P distinct base streams built to reach the
frontend's edges; the oracle runs over the P base streams only."""

import os

import numpy as np
import pytest

import oracle
from conftest import GOLDEN
from test_g711 import ulaw_ref
from test_gpu_frontend_full_size import check_features, check_state, features_call, oracle_state, stress_audio
from test_gpu_full_size import check_streams, periodic_streams

pytestmark = pytest.mark.gpu

P = 257
N = 96000                      # two calls of 48 000 samples: 298 rows, then 300 entering with 320 carried samples
CALLS = ((0, 48000, 0, 298), (48000, 96000, 298, 300))


class Inputs:
    def __init__(self, torch):
        self.torch = torch
        self.base = stress_audio()[:P]
        self.want, _ = oracle.run_pipeline(None, self.base, want_probs=False, threads=8)
        self.state = oracle_state(self.base)
        self.dev = periodic_streams(torch, self.base, 65536, ())


@pytest.fixture(scope="module")
def inputs(torch_cuda):
    return Inputs(torch_cuda)


def _wave(torch):
    return 4 * torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("count", ["12 x SMs", "12 x SMs + 1", "65509"])
def test_stream_counts_over_two_calls(inputs, count):
    from microwakeword_b200.engine import StreamEngine
    torch = inputs.torch
    wave = _wave(torch)
    S = {"12 x SMs": 3 * wave, "12 x SMs + 1": 3 * wave + 1, "65509": 65509}[count]
    eng = StreamEngine(None, n_streams=S)
    for lo, hi, row, T in CALLS:
        out = features_call(eng, inputs.dev[:S, lo:hi].contiguous(), 2)           # the fused clip kernel + the carry update
        assert out.shape == (S, T, 40)
        check_features(torch, out, inputs.want[:, row:row + T], (count, lo))
        del out
    check_state(eng.state_dict(), inputs.state, count)


@pytest.mark.parametrize("kind", ["f32", "ulaw"])
def test_float32_and_ulaw_clips_equal_an_int16_twin(inputs, kind):
    """12 x SMs + 7 streams; the mu-law side takes codes of the audio, its twin their int16 decoding (and the oracle the same)"""
    from microwakeword_b200.engine import StreamEngine
    torch = inputs.torch
    S = 3 * _wave(torch) + 7
    if kind == "ulaw":
        codes = np.random.default_rng(5).integers(0, 256, (P, N), dtype=np.uint8)
        dec = ulaw_ref(codes)
        want, _ = oracle.run_pipeline(None, dec, want_probs=False, threads=8)
        codes_dev = periodic_streams(torch, codes, S, ())
        dec_dev = periodic_streams(torch, dec, S, ())
    else:
        want, dec_dev = inputs.want, inputs.dev[:S]
    side, twin = StreamEngine(None, n_streams=S), StreamEngine(None, n_streams=S)
    for lo, hi, row, T in CALLS:
        x16 = dec_dev[:, lo:hi].contiguous()
        if kind == "ulaw":
            a = side.features(codes_dev[:, lo:hi].contiguous(), law="ulaw")
        else:
            a = side.features(x16.to(torch.float32).mul_(1.0 / 32768))           # exact: to_int16 gives x16 back
        b = twin.features(x16)
        assert torch.equal(a, b), (kind, lo)
        check_features(torch, a, want[:, row:row + T], (kind, lo))
        del a, b
    st_a, st_b = side.state_dict(), twin.state_dict()
    for k in ("carry", "estimate", "frontend_buffered"):
        assert np.array_equal(np.asarray(st_a[k]), np.asarray(st_b[k])), k
    if kind == "f32":
        check_state(st_a, inputs.state, kind)


def test_stream_tiles_with_a_last_tile_below_one_wave(inputs, monkeypatch):
    """MWW_SCRATCH_MB=16: predict_clip's feature scratch holds 703 streams of 298 rows, so 3 x 703 + 4 x SMs - 1 streams make
    three full tiles and a last one of 4 x SMs - 1 streams (then 699-stream tiles for the 300-row call).  Probabilities
    bit-identical to an untiled engine's and to the oracle's, state equal to both."""
    from microwakeword_b200.engine import StreamEngine
    torch = inputs.torch
    wave = _wave(torch)
    tile = (16 << 20) // (298 * 40 * 2)
    assert tile >= wave
    S = 3 * tile + wave - 1
    with open(os.path.join(GOLDEN, "okay_nabu_synth_int8.mww"), "rb") as f:
        blob = f.read()
    plain = StreamEngine(blob, n_streams=S)
    monkeypatch.setenv("MWW_SCRATCH_MB", "16")                    # read at mww_create
    tiled = StreamEngine(blob, n_streams=S)
    got = []
    for lo, hi, _, _ in CALLS:
        x = inputs.dev[:S, lo:hi].contiguous()
        l0 = tiled.launch_count
        a = tiled.predict_clip(x)
        assert tiled.launch_count - l0 >= 2 * 4, "the call was not tiled"
        b = plain.predict_clip(x)
        assert torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32)), ("tiled != untiled", lo)
        got.append(a)
    _, want = oracle.run_pipeline(blob, inputs.base, want_features=False, threads=8)
    check_streams(torch, torch.cat(got, 1), want, True, "tiled int8")
    st_t, st_p = tiled.state_dict(), plain.state_dict()
    for k in st_p:
        assert np.array_equal(np.asarray(st_t[k]), np.asarray(st_p[k])), k
    check_state(st_t, inputs.state, "tiled")
