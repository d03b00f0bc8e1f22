"""Audio at 8, 22.05, 24, 32, 44.1 and 48 kHz through the GPU resampler in front of the frontend (run with -m gpu on an H100).

The contract (include/mww.h, mww_set_input_rate): a handle at input rate r given audio x computes exactly what a 16 kHz
handle computes given the integer resampling of x (tests/resample_oracle.py, scipy's upfirdn over the library's own taps,
the rounding shift, int16 saturation) -- features, fp32 and int8 probabilities bit for bit -- on the device, host and
remote-from-host paths, with int16 and float32 input, under any split of the audio into calls, in 30 ms live calls, on
multi-model handles with stream sets and in many small tiles.  Resets, state round trips and refusals behave as stated."""

import ctypes
import os

import numpy as np
import pytest

import resample_oracle as ref
from conftest import GOLDEN
from microwakeword_b200 import _lib
from microwakeword_b200.audio.audio_utils import to_int16
from microwakeword_b200.engine import MultiModelEngine, StreamEngine

pytestmark = pytest.mark.gpu

F32 = os.path.join(GOLDEN, "okay_nabu_synth_f32.mww")
I8 = os.path.join(GOLDEN, "okay_nabu_synth_int8.mww")
S = 6


def _taps(rate):
    L = _lib.lib()
    n = ctypes.c_int()
    assert L.mww_resample_taps(rate, None, 0, ctypes.byref(n), None, None) == 0
    out = np.zeros(n.value, np.int32)
    assert L.mww_resample_taps(rate, out.ctypes.data, out.size, None, None, None) == 0
    return out


def oracle16(x, rate):
    """float32 or int16 host audio [S, N] at `rate` -> the int16 16 kHz audio a 16 kHz handle is given instead"""
    if x.dtype == np.float32:
        with np.errstate(invalid="ignore", over="ignore"):
            x = to_int16(x)
    return ref.resample(x, _taps(rate), rate)


def make_audio(rate, n_streams, n, seed, dtype):
    rng = np.random.default_rng(seed)
    amp = (10.0 ** rng.uniform(-3.0, 0.2, n_streams)).astype(np.float32)[:, None]     # -60 dBFS .. clipping
    t = np.arange(n, dtype=np.float32) / rate
    tone = np.sin(2 * np.pi * rng.uniform(100, rate / 2, (n_streams, 1)).astype(np.float32) * t)
    x = ((rng.standard_normal((n_streams, n), dtype=np.float32) * 0.5 + tone) * amp).astype(np.float32)
    if dtype == np.float32:
        return x
    with np.errstate(invalid="ignore", over="ignore"):
        return to_int16(x)


def dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def feats(e, x):
    return e.features(dev(x)).cpu().numpy().copy()


@pytest.mark.parametrize("dtype", [np.int16, np.float32], ids=["int16", "float32"])
@pytest.mark.parametrize("rate", ref.RATES)
def test_paths_equal_16k_handle_on_oracle_audio(torch_cuda, rate, dtype):
    x = make_audio(rate, S, rate + 777, rate + 1, dtype)
    x16 = oracle16(x, rate)
    assert np.array_equal(feats(StreamEngine(None, S, 0, input_rate=rate), x), feats(StreamEngine(None, S, 0), x16))
    for blob in (F32, I8):
        want = StreamEngine(blob, S, 0).predict_clip(dev(x16)).cpu().numpy()
        got = StreamEngine(blob, S, 0, input_rate=rate).predict_clip(dev(x)).cpu().numpy()
        assert got.shape == want.shape and np.array_equal(got, want), (blob, "device")
        host = StreamEngine(blob, S, 0, input_rate=rate).predict_clip_host(x)
        assert np.array_equal(host, want), (blob, "host")
        e = StreamEngine(blob, S, 0, input_rate=rate)
        buf = e.host_buffer(x.shape, x.dtype)
        buf[:] = x
        remote = e.predict_clip_remote(buf.ctypes.data, x.shape[1], dtype=x.dtype).cpu().numpy()
        assert np.array_equal(remote, want), (blob, "remote")


@pytest.mark.parametrize("rate", ref.RATES)
def test_random_call_splits_equal_one_call(torch_cuda, rate):
    rng = np.random.default_rng(rate)
    N = rate // 2 + 311
    x = make_audio(rate, S, N, rate + 2, np.int16)
    one_f = feats(StreamEngine(None, S, 0, input_rate=rate), x)
    one_p = StreamEngine(I8, S, 0, input_rate=rate).predict_clip(dev(x)).cpu().numpy()
    fe, e = StreamEngine(None, S, 0, input_rate=rate), StreamEngine(I8, S, 0, input_rate=rate)
    got_f, got_p, pos = [], [], 0
    while pos < N:
        n = min(N - pos, int(rng.choice([0, 1, 2, 440, 441, 442, int(rng.integers(1, 9000))])))
        chunk = x[:, pos:pos + n]
        got_f.append(feats(fe, chunk))
        got_p.append(e.predict_clip(dev(chunk)).cpu().numpy())
        pos += n
    assert np.array_equal(np.concatenate(got_f, 1), one_f)
    assert np.array_equal(np.concatenate(got_p, 1), one_p)
    rate_now, seen = e._rate()
    assert (rate_now, seen) == (rate, N)


@pytest.mark.parametrize("rate", [r for r in ref.RATES if r * 3 % 100 == 0])
def test_live_calls_equal_16k_live_calls_and_take_live_kernels(torch_cuda, rate):
    n = rate * 3 // 100                       # 30 ms: 480 samples at 16 kHz
    calls = 24
    x = make_audio(rate, S, n * calls, rate + 3, np.float32)
    x16 = oracle16(x, rate)
    for blob in (F32, I8):
        e, base = StreamEngine(blob, S, 0, input_rate=rate), StreamEngine(blob, S, 0)
        live, want, per_call, per_call16 = [], [], [], []
        for i in range(calls):
            c0, b0 = e.launch_count, base.launch_count
            live.append(e.step(dev(x[:, i * n:(i + 1) * n])).cpu().numpy())
            want.append(base.step(dev(x16[:, i * 480:(i + 1) * 480])).cpu().numpy())
            per_call.append(e.launch_count - c0)
            per_call16.append(base.launch_count - b0)
        assert np.array_equal(np.concatenate(live, 1), np.concatenate(want, 1)), blob
        if blob == I8:                        # int8: live and clip kernels agree bit for bit, so live calls equal one clip call
            clip = StreamEngine(blob, S, 0, input_rate=rate).predict_clip(dev(x)).cpu().numpy()
            assert np.array_equal(np.concatenate(live, 1), clip)
        # every call: the 16 kHz live call's launches (fused frontend + live-step NN once rows flow) plus the resampler
        assert per_call == [c + 1 for c in per_call16], (per_call, per_call16)
        assert max(per_call16[4:]) <= 2


def test_multi_model_stream_sets_in_small_tiles(torch_cuda, monkeypatch):
    monkeypatch.setenv("MWW_SCRATCH_MB", "1")
    monkeypatch.setenv("MWW_MIN_TILE_STREAMS", "1")
    n_streams, rate = 40, 44100
    sets = [None, list(range(1, n_streams, 3))]
    x = make_audio(rate, n_streams, rate + 5, 7, np.float32)
    x16 = oracle16(x, rate)
    want = MultiModelEngine([F32, I8], n_streams, 0, streams=sets).predict_clip(dev(x16))
    got = MultiModelEngine([F32, I8], n_streams, 0, streams=sets, input_rate=rate).predict_clip(dev(x))
    host = MultiModelEngine([F32, I8], n_streams, 0, streams=sets, input_rate=rate).predict_clip_host(x)
    for k in range(2):
        assert np.array_equal(got[k].cpu().numpy(), want[k].cpu().numpy()), k
        assert np.array_equal(host[k], want[k].cpu().numpy()), k
    # a second call continues from the carried history in every tile
    y = make_audio(rate, n_streams, 4410, 8, np.float32)
    both16 = oracle16(np.concatenate([x, y], 1), rate)[:, x16.shape[1]:]
    e16 = MultiModelEngine([F32, I8], n_streams, 0, streams=sets)
    e16.predict_clip(dev(x16))
    e = MultiModelEngine([F32, I8], n_streams, 0, streams=sets, input_rate=rate)
    e.predict_clip_host(x)
    a, b = e.predict_clip_host(y), e16.predict_clip(dev(both16))
    for k in range(2):
        assert np.array_equal(a[k], b[k].cpu().numpy()), k


def test_bench_shape_48k(torch_cuda):
    torch = torch_cuda
    n_streams, rate, N = 65536, 48000, 3 * 48000
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randint(-12000, 12000, (n_streams, N), dtype=torch.int16, device="cuda", generator=g)
    f = StreamEngine(None, n_streams, 0, input_rate=rate).features(x)
    pick = np.array([0, 1, 2047, 2048, 30000, 32767, 32768, 50001, 65534, 65535])
    x16 = oracle16(x[torch.from_numpy(pick).cuda()].cpu().numpy(), rate)
    want = feats(StreamEngine(None, pick.size, 0), x16)
    got = f.view(torch.int16)[torch.from_numpy(pick).cuda()].cpu().numpy().view(np.uint16)
    assert np.array_equal(got, want)


def test_resets_and_state_round_trip(torch_cuda):
    rate = 44100
    e = StreamEngine(F32, 4, 0, input_rate=rate)
    x = make_audio(rate, 4, 5000, 11, np.int16)
    y = make_audio(rate, 4, 3000, 12, np.int16)
    e.predict_clip(dev(x))
    st = e.state_dict()
    assert st["input_rate"] == rate and st["inputs_seen"] == 5000 and st["resampler_history"].shape == (4, e.resampler_history())
    assert np.array_equal(st["resampler_history"], x[:, -e.resampler_history():])
    p1 = e.predict_clip(dev(y)).cpu().numpy()
    e.load_state_dict(st)
    assert e._rate() == (rate, 5000)
    assert np.array_equal(e.predict_clip(dev(y)).cpu().numpy(), p1)
    # reset by id: those streams' history only; the counter stays
    e.reset([1, 3])
    st2 = e.state_dict()
    assert st2["inputs_seen"] == 8000
    assert not st2["resampler_history"][[1, 3]].any()
    assert np.array_equal(st2["resampler_history"][[0, 2]], y[[0, 2], -e.resampler_history():])
    # reset_frontend: history and counter zero -- the next call equals a fresh handle's
    fe = StreamEngine(None, 4, 0, input_rate=rate)
    fe.features(dev(x))
    fe.reset_frontend()
    assert fe._rate() == (rate, 0)
    assert np.array_equal(feats(fe, y), feats(StreamEngine(None, 4, 0, input_rate=rate), y))
    fe.features(dev(x))
    fe.reset()
    assert fe._rate() == (rate, 0)
    assert np.array_equal(feats(fe, y), feats(StreamEngine(None, 4, 0, input_rate=rate), y))


def test_refusals_leave_the_handle_unchanged(torch_cuda):
    e = StreamEngine(I8, 4, 0, input_rate=48000)
    with pytest.raises(_lib.MwwError) as r:
        e.set_input_rate(11025)
    assert r.value.code == -5 and e.input_rate == 48000
    x = make_audio(48000, 4, 1000, 13, np.int16)
    e.predict_clip(dev(x))
    before = e.state_dict()
    with pytest.raises(_lib.MwwError) as r:
        e.set_input_rate(16000)
    assert r.value.code == -1 and e.input_rate == 48000
    with pytest.raises(_lib.MwwError) as r:
        e.export_streams([0, 1])
    assert r.value.code == -5
    recs = StreamEngine(I8, 4, 0).export_streams([0, 1])
    with pytest.raises(_lib.MwwError) as r:
        e.import_streams([2, 3], recs)
    assert r.value.code == -5
    after = e.state_dict()
    for k in before:
        assert np.array_equal(np.asarray(before[k]), np.asarray(after[k])), k
    # after a reset the rate may change again, and 16 kHz is the plain path again
    e.reset()
    e.set_input_rate(16000)
    assert e.input_rate == 16000 and "resampler_history" not in e.state_dict()
