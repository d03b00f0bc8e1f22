"""Per-stream input rates (mww_set_stream_rates) on the GPU (run with -m gpu on an H100).

The contract (include/mww.h): stream s of a handle with per-stream rates is bit-identical to a stream of a handle at the
single rate r_s (a plain 16 kHz handle when r_s = 16000) given the same D_s samples in every call -- features, fp32 and
int8 probabilities, state and resampler history -- on the device, host (pinned and pageable) and remote-from-host paths,
with int16 and float32 input, under any even split into calls, in 30 ms live calls, on multi-model handles with stream sets
in small tiles, across rate changes, resets and state round trips, and at 65 536 streams.  Every comparison below is
against such single-rate handles."""

import os

import numpy as np
import pytest

from conftest import GOLDEN
from microwakeword_b200 import _lib
from microwakeword_b200.audio.audio_utils import to_int16
from microwakeword_b200.engine import (INPUT_RATES, RATE_PER_STREAM, MultiModelEngine, StreamEngine, inputs_for_rates, rate_inputs,
                                       resampler_history_len)

pytestmark = pytest.mark.gpu

F32 = os.path.join(GOLDEN, "okay_nabu_synth_f32.mww")
I8 = os.path.join(GOLDEN, "okay_nabu_synth_int8.mww")
RATES14 = np.array([48000, 8000, 16000, 44100, 22050, 24000, 32000, 16000, 48000, 22050, 8000, 44100, 32000, 24000], np.int32)


def dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def host(x):
    return x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)


def make_streams(rates, total16, seed, dtype):
    """per stream its whole input at its own rate: N(total16, r_s) samples (a list of 1-D arrays)"""
    rng = np.random.default_rng(seed)
    out = []
    for r in rates:
        n = rate_inputs(total16, int(r))
        t = np.arange(n, dtype=np.float32) / r
        x = (rng.standard_normal(n).astype(np.float32) * 0.3 + np.sin(2 * np.pi * rng.uniform(100, r / 2) * t)) * rng.uniform(0.01, 1.2)
        x = x.astype(np.float32)
        if dtype == np.int16:
            with np.errstate(invalid="ignore", over="ignore"):
                x = to_int16(x)
        out.append(x)
    return out


def call_rows(streams, rates, t, n16, extra=0):
    """[S, max D_s + extra] rows of a call of n16 at counter t (padding past D_s is garbage the library must not read)"""
    D = inputs_for_rates(rates, t, n16)
    x = np.full((len(streams), int(D.max()) + extra if len(streams) else 0), 7, streams[0].dtype)
    for s, r in enumerate(rates):
        a = rate_inputs(t, int(r))
        x[s, :D[s]] = streams[s][a:a + D[s]]
    return x, D


class Refs:
    """one single-rate engine per rate over that rate's streams; results assembled in stream order"""

    def __init__(self, blob, rates):
        self.rates = np.asarray(rates)
        self.ids = {int(r): np.flatnonzero(self.rates == r) for r in np.unique(self.rates)}
        self.eng = {r: StreamEngine(blob, ids.size, 0, input_rate=r) for r, ids in self.ids.items()}

    def run(self, x, D, what):
        parts = {}
        for r, ids in self.ids.items():
            rows = np.ascontiguousarray(x[ids, :D[ids[0]]])
            e = self.eng[r]
            parts[r] = host(e.features(dev(rows)) if what == "features" else e.predict_clip(dev(rows)))
        shape = next(iter(parts.values())).shape[1:]
        out = np.zeros((self.rates.size,) + shape, next(iter(parts.values())).dtype)
        for r, ids in self.ids.items():
            out[ids] = parts[r]
        return out

    def state(self, s):
        """stream s's state in its reference engine: carry, estimate, nn, pending and resampler history"""
        r = int(self.rates[s])
        j = int(np.flatnonzero(self.ids[r] == s)[0])
        d = self.eng[r].state_dict()
        hist = d["resampler_history"][j] if "resampler_history" in d else np.zeros(0, np.int16)
        return {k: d[k][j] for k in ("carry", "estimate", "nn", "pending") if k in d}, hist


def assert_state_equal(e, refs):
    d = e.state_dict()
    assert d["input_rate"] == RATE_PER_STREAM and np.array_equal(d["stream_rates"], refs.rates)
    for s in range(refs.rates.size):
        want, hist = refs.state(s)
        for k, v in want.items():
            assert np.array_equal(d[k][s], v), (s, k)
        assert np.array_equal(d["resampler_history"][s, :hist.size], hist), s


@pytest.mark.parametrize("dtype", [np.int16, np.float32], ids=["int16", "float32"])
def test_all_rates_one_handle_every_path(torch_cuda, dtype):
    rates, n16 = RATES14, 24000
    streams = make_streams(rates, n16, 1, dtype)
    x, D = call_rows(streams, rates, 0, n16, extra=5)
    fe = StreamEngine(None, rates.size, 0, stream_rates=rates)
    assert np.array_equal(host(fe.features(dev(x), samples16=n16)), Refs(None, rates).run(x, D, "features"))
    for blob in (F32, I8):
        refs = Refs(blob, rates)
        want = refs.run(x, D, "predict")
        e = StreamEngine(blob, rates.size, 0, stream_rates=rates)
        assert np.array_equal(host(e.predict_clip(dev(x), samples16=n16)), want), (blob, "device")
        assert_state_equal(e, refs)
        pageable = StreamEngine(blob, rates.size, 0, stream_rates=rates).predict_clip_host(x, samples16=n16)
        assert np.array_equal(pageable, want), (blob, "host pageable")
        e = StreamEngine(blob, rates.size, 0, stream_rates=rates)
        buf = e.host_buffer(x.shape, x.dtype)
        buf[:] = x
        assert np.array_equal(e.predict_clip_host(buf, samples16=n16), want), (blob, "host pinned")
        e = StreamEngine(blob, rates.size, 0, stream_rates=rates)
        got = e.predict_clip_remote(buf.ctypes.data, x.shape[1], dtype=x.dtype, samples16=n16, tiles=3)
        assert np.array_equal(host(got), want), (blob, "remote")


def test_random_even_splits_and_live_calls(torch_cuda):
    rng = np.random.default_rng(3)
    rates = RATES14
    total = 2 * 9000
    streams = make_streams(rates, total, 4, np.int16)
    x, D = call_rows(streams, rates, 0, total)
    one = StreamEngine(I8, rates.size, 0, stream_rates=rates).predict_clip(dev(x), samples16=total).cpu().numpy()
    e, t, got = StreamEngine(I8, rates.size, 0, stream_rates=rates), 0, []
    while t < total:
        n16 = min(total - t, 2 * int(rng.choice([0, 1, 240, 241, int(rng.integers(1, 3000))])))
        xc, _ = call_rows(streams, rates, t, n16)
        assert np.array_equal(e.inputs_for(n16), inputs_for_rates(rates, t, n16))
        got.append(e.predict_clip(dev(xc), samples16=n16).cpu().numpy())
        t += n16
    assert np.array_equal(np.concatenate(got, 1), one)
    assert e._rate() == (RATE_PER_STREAM, total)
    # 30 ms live calls: n16 = 480 at every rate (22.05 kHz alternates 661 / 662 samples), fp32 and int8
    calls = 30
    streams = make_streams(rates, 480 * calls, 5, np.float32)
    for blob in (F32, I8):
        e, refs, live, want = StreamEngine(blob, rates.size, 0, stream_rates=rates), Refs(blob, rates), [], []
        for i in range(calls):
            xc, Dc = call_rows(streams, rates, 480 * i, 480)
            live.append(host(e.step(dev(xc))))
            want.append(refs.run(xc, Dc, "predict"))
        assert np.array_equal(np.concatenate(live, 1), np.concatenate(want, 1)), blob
        assert_state_equal(e, refs)


def test_multi_model_stream_sets_in_small_tiles(torch_cuda, monkeypatch):
    monkeypatch.setenv("MWW_SCRATCH_MB", "1")
    monkeypatch.setenv("MWW_MIN_TILE_STREAMS", "1")
    n_streams = 40
    rates = np.array([INPUT_RATES[(s * 5 + s // 7) % 7] for s in range(n_streams)], np.int32)
    sets = [None, list(range(1, n_streams, 3))]
    n16 = 16000
    streams = make_streams(rates, 2 * n16, 7, np.float32)
    e = MultiModelEngine([F32, I8], n_streams, 0, streams=sets, stream_rates=rates)
    eh = MultiModelEngine([F32, I8], n_streams, 0, streams=sets, stream_rates=rates)
    refs = [Refs(F32, rates), Refs(I8, rates)]
    for c in range(2):
        x, D = call_rows(streams, rates, c * n16, n16, extra=3)
        got, got_h = e.predict_clip(dev(x), samples16=n16), eh.predict_clip_host(x, samples16=n16)
        for k in range(2):
            want = refs[k].run(x, D, "predict")
            if sets[k] is not None:
                want = want[sets[k]]
            assert np.array_equal(host(got[k]), want), (c, k)
            assert np.array_equal(got_h[k], want), (c, k)


def _restart(blob, st, s, rate, t):
    """a one-stream engine at `rate` holding stream s's frontend and NN state from state_dict `st`, its resampler history
    zeroed at counter t (what a rate change leaves a stream)"""
    ref = StreamEngine(blob, 1, 0, input_rate=rate)
    d = {k: st[k][[s]] for k in ("carry", "estimate", "nn", "pending") if k in st}
    d.update(frontend_buffered=st["frontend_buffered"], pending_rows=st["pending_rows"], input_rate=rate)
    if rate != 16000:
        d.update(resampler_history=np.zeros((1, resampler_history_len(rate)), np.int16), inputs_seen=rate_inputs(t, rate))
    ref.load_state_dict(d)
    return ref


def test_rate_changes_mid_stream(torch_cuda):
    rates = RATES14.copy()
    n16 = 9600
    for blob in (F32, I8):
        streams = make_streams(rates, n16, 8, np.int16)
        e, refs = StreamEngine(blob, rates.size, 0, stream_rates=rates), Refs(blob, rates)
        x, D = call_rows(streams, rates, 0, n16)
        assert np.array_equal(host(e.predict_clip(dev(x), samples16=n16)), refs.run(x, D, "predict"))
        st = e.state_dict()
        change = {0: 8000, 2: 44100, 5: 16000, 9: 22050}          # 9 keeps its rate: its history is zeroed all the same
        new = rates.copy()
        for s, r in change.items():
            new[s] = r
        e.set_stream_rates(list(change), list(change.values()))
        assert np.array_equal(e.stream_rates, new)
        after = e.state_dict()
        for s in range(rates.size):
            if s in change:
                assert not after["resampler_history"][s].any(), s
            else:
                assert np.array_equal(after["resampler_history"][s], st["resampler_history"][s]), s
            for k in ("carry", "estimate", "nn", "pending"):
                assert np.array_equal(after[k][s], st[k][s]), (s, k)
        restarted = {s: _restart(blob, st, s, r, n16) for s, r in change.items()}
        streams2 = make_streams(new, 3 * n16, 9, np.int16)
        for c in (1, 2):
            x, D = call_rows(streams2, new, c * n16, n16)
            got = host(e.predict_clip(dev(x), samples16=n16))
            # the unchanged streams continue on their references (rows cut at each reference's own rate)
            want = refs.run(x, inputs_for_rates(rates, c * n16, n16), "predict")
            for s in range(rates.size):
                if s in change:
                    w = host(restarted[s].predict_clip(dev(x[[s], :D[s]])))[0]
                else:
                    w = want[s]
                assert np.array_equal(got[s], w), (blob, c, s)


def test_resets_state_round_trip_and_leaving_the_mode(torch_cuda):
    rates = RATES14
    n16 = 6400
    streams = make_streams(rates, 4 * n16, 10, np.int16)
    e = StreamEngine(F32, rates.size, 0, stream_rates=rates)
    x1, _ = call_rows(streams, rates, 0, n16)
    x2, _ = call_rows(streams, rates, n16, n16)
    e.predict_clip(dev(x1), samples16=n16)
    st = e.state_dict()
    assert st["inputs_seen"] == n16 and st["resampler_history"].shape == (rates.size, 243)
    p2 = host(e.predict_clip(dev(x2), samples16=n16))
    e2 = StreamEngine(F32, rates.size, 0)                        # a fresh 16 kHz engine takes the mode from the state
    e2.load_state_dict(st)
    e.load_state_dict(st)
    assert e._rate() == e2._rate() == (RATE_PER_STREAM, n16)
    assert np.array_equal(host(e.predict_clip(dev(x2), samples16=n16)), p2)
    assert np.array_equal(host(e2.predict_clip(dev(x2), samples16=n16)), p2)
    # reset by id: those streams' histories (and frontend / models); the counter and the rates stay
    e.reset([1, 3])
    d = e.state_dict()
    assert d["inputs_seen"] == 2 * n16 and np.array_equal(d["stream_rates"], rates)
    assert not d["resampler_history"][[1, 3]].any() and d["resampler_history"][[0, 4]].any()
    # full reset and reset_frontend: every history and the counter zero, rates kept; the next call equals a fresh engine's
    for how in ("reset", "reset_frontend"):
        f = StreamEngine(None, rates.size, 0, stream_rates=rates)
        f.features(dev(x1), samples16=n16)
        getattr(f, how)()
        assert f._rate() == (RATE_PER_STREAM, 0) and np.array_equal(f.stream_rates, rates)
        assert not f.state_dict()["resampler_history"].any()
        fresh = StreamEngine(None, rates.size, 0, stream_rates=rates)
        assert np.array_equal(host(f.features(dev(x1), samples16=n16)), host(fresh.features(dev(x1), samples16=n16))), how
    # set_input_rate at counter 0 leaves the mode: one rate for every stream again, exactly a fresh engine at that rate
    f.reset()
    f.set_input_rate(48000)
    assert f.input_rate == 48000 and set(f.stream_rates.tolist()) == {48000}
    y = make_streams([48000] * rates.size, 4800, 11, np.int16)
    y = np.stack(y)
    assert np.array_equal(host(f.features(dev(y))), host(StreamEngine(None, rates.size, 0, input_rate=48000).features(dev(y))))
    f.reset()
    f.set_input_rate(16000)
    assert f.input_rate == 16000 and "resampler_history" not in f.state_dict()


def test_refusals_leave_the_handle_unchanged(torch_cuda):
    import ctypes
    rates = RATES14
    e = StreamEngine(I8, rates.size, 0, stream_rates=rates)
    streams = make_streams(rates, 4000, 12, np.int16)
    x, D = call_rows(streams, rates, 0, 2000)
    e.predict_clip(dev(x), samples16=2000)
    before = e.state_dict()
    L, h = e._L, e._h
    ids = np.array([0, 1], np.int32)

    def refused(code, fn, *args):
        assert fn(*args) == code
    refused(-5, L.mww_set_stream_rates, h, ids.ctypes.data, np.array([8000, 11025], np.int32).ctypes.data, 2, None)
    refused(-1, L.mww_set_stream_rates, h, np.array([0, 14], np.int32).ctypes.data, np.array([8000, 8000], np.int32).ctypes.data, 2, None)
    refused(-1, L.mww_set_stream_rates, h, np.array([3, 3], np.int32).ctypes.data, np.array([8000, 8000], np.int32).ctypes.data, 2, None)
    refused(-1, L.mww_set_stream_rates, h, ids.ctypes.data, ids.ctypes.data, -1, None)
    x2, D2 = call_rows(streams, rates, 2000, 2000)
    xd = dev(x2)
    probs = np.zeros((rates.size, 64), np.float32)
    got = ctypes.c_int()
    refused(-1, L.mww_predict_clip, h, xd.data_ptr(), 1999, xd.stride(0), dev(probs).data_ptr(), 64, ctypes.byref(got), None)   # odd n16
    refused(-1, L.mww_predict_clip, h, xd.data_ptr(), 2000, int(D2.max()) - 1, dev(probs).data_ptr(), 64, ctypes.byref(got), None)
    refused(-1, L.mww_predict_clip_host, h, x2.ctypes.data, 2000, int(D2.max()) - 1, probs.ctypes.data, 64, ctypes.byref(got))
    refused(-1, L.mww_set_resampler_state, h, None, 2001)
    with pytest.raises(_lib.MwwError) as r:
        e.set_input_rate(16000)                                  # counter not 0
    assert r.value.code == -1
    with pytest.raises(_lib.MwwError) as r:
        e.export_streams([0, 1])
    assert r.value.code == -5
    recs = StreamEngine(I8, rates.size, 0).export_streams([0, 1])
    with pytest.raises(_lib.MwwError) as r:
        e.import_streams([2, 3], recs)
    assert r.value.code == -5
    with pytest.raises(ValueError):
        e.predict_clip(dev(x2), samples16=1999)
    with pytest.raises(ValueError):
        e.predict_clip(dev(x2[:, :100]), samples16=2000)
    with pytest.raises(ValueError):
        e.predict_clip(dev(x2))
    after = e.state_dict()
    for k in before:
        assert np.array_equal(np.asarray(before[k]), np.asarray(after[k])), k
    rate, seen = ctypes.c_int(), ctypes.c_longlong()
    assert L.mww_get_input_rate(h, ctypes.byref(rate), ctypes.byref(seen)) == 0 and (rate.value, seen.value) == (RATE_PER_STREAM, 2000)
    # the first call needs an empty 16 kHz handle
    busy = StreamEngine(None, 4, 0)
    busy.features(dev(np.zeros((4, 100), np.int16)))
    with pytest.raises(_lib.MwwError) as r:
        busy.set_stream_rates([0], [8000])
    assert r.value.code == -1 and busy.input_rate == 16000
    with pytest.raises(_lib.MwwError) as r:
        StreamEngine(None, 4, 0, input_rate=48000).set_stream_rates([0], [8000])
    assert r.value.code == -1


def test_65536_streams_every_rate(torch_cuda):
    torch = torch_cuda
    S = 65536
    rates = np.array([INPUT_RATES[s % 7] for s in range(S)], np.int32)
    pick = np.array([0, 1, 2, 3, 4, 5, 6, 2047, 2048, 30000, 32767, 32768, 50001, 65534, 65535])
    g = torch.Generator(device="cuda").manual_seed(6)
    # one 3 s call
    n16 = 48000
    D = inputs_for_rates(rates, 0, n16)
    x = torch.randint(-12000, 12000, (S, int(D.max())), dtype=torch.int16, device="cuda", generator=g)
    f = StreamEngine(None, S, 0, stream_rates=rates).features(x, samples16=n16)
    xp = x[torch.from_numpy(pick).cuda()].cpu().numpy()
    want = Refs(None, rates[pick]).run(xp, D[pick], "features")
    assert np.array_equal(f.view(torch.int16)[torch.from_numpy(pick).cuda()].cpu().numpy().view(np.uint16), want)
    del x, f
    # 100 live calls
    e, refs, got, want = StreamEngine(I8, S, 0, stream_rates=rates), Refs(I8, rates[pick]), [], []
    idx = torch.from_numpy(pick).cuda()
    for i in range(100):
        D = inputs_for_rates(rates, 480 * i, 480)
        xc = torch.randint(-12000, 12000, (S, int(D.max())), dtype=torch.int16, device="cuda", generator=g)
        got.append(e.step(xc)[idx].cpu().numpy())
        want.append(refs.run(xc[idx].cpu().numpy(), D[pick], "predict"))
    assert np.array_equal(np.concatenate(got, 1), np.concatenate(want, 1))
