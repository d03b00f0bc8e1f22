"""Per-stream sample formats (mww_set_stream_formats, the _mixed entry points) on the GPU (run with -m gpu on an H100).

The method is the twin handle: the same models and rates, fed each stream's bytes decoded to int16 by this file's own
oracle (tests/test_g711.py's NumPy statement of the G.711 rule, the float32 conversion of audio_utils.to_int16).  The mixed
handle must give bit-identical probabilities, features, full state (resampler history included) and audio history, on the
device, host (pinned, pageable, write-combined) and remote paths, in live 30 ms calls and 3 s calls over several tiles, with
formats changed between calls, for StreamEngine and MultiModelEngine with stream sets, fp32 and int8 models, at 65 536
streams, and across stream moves.  Refusals leave the handle bit-identical."""

import ctypes
import os

import numpy as np
import pytest

from conftest import GOLDEN
from microwakeword_b200 import _lib
from microwakeword_b200.engine import (INPUT_RATES, SAMPLE_FORMATS, MultiModelEngine, StreamEngine, StreamRecords, bytes_for_formats,
                                       inputs_for_rates)
from test_stream_formats import decode, mixed_rows, samples

pytestmark = pytest.mark.gpu

F32 = os.path.join(GOLDEN, "okay_nabu_synth_f32.mww")
I8 = os.path.join(GOLDEN, "okay_nabu_synth_int8.mww")
S16, ULAW, ALAW, F32F = (SAMPLE_FORMATS[k] for k in ("s16", "ulaw", "alaw", "f32"))
RATES16 = np.array([8000, 8000, 48000, 16000, 44100, 22050, 24000, 32000, 8000, 48000, 16000, 22050, 8000, 44100, 32000, 24000], np.int32)
FMTS16 = np.array([ULAW, ALAW, F32F, S16, S16, ULAW, F32F, ALAW, S16, F32F, ULAW, ALAW, F32F, ULAW, S16, ALAW], np.int32)


def dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def host(x):
    return x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)


def call(rng, rates, fmts, t, n16, pad=0xA5):
    """one call's mixed rows (uint8, pitch a multiple of 4) and the twin's int16 rows of the same samples decoded"""
    D = inputs_for_rates(rates, t, n16)
    parts = [samples(rng, int(D[s]), int(fmts[s])) for s in range(len(rates))]
    pitch = max((int(bytes_for_formats(rates, fmts, t, n16).max()) + 3) // 4 * 4, 4)
    x = mixed_rows(parts, pitch, pad)
    y = np.zeros((len(rates), max(int(D.max()), 1)), np.int16)
    for s, p in enumerate(parts):
        y[s, :p.size] = decode(p, int(fmts[s]))
    return x, y


def engines(cls, blob, rates, fmts, history=0, **kw):
    """(mixed engine, int16 twin) over the same rates"""
    a = cls(blob, len(rates), 0, stream_rates=rates, stream_formats=fmts, **kw)
    b = cls(blob, len(rates), 0, stream_rates=rates, **kw)
    if history:
        a.set_audio_history(history)
        b.set_audio_history(history)
    return a, b


def same_state(a, b, where="state"):
    if isinstance(a, dict):
        keys = set(a) - {"stream_formats"}
        assert keys == set(b) - {"stream_formats"}, where
        for k in keys:
            same_state(a[k], b[k], "%s.%s" % (where, k))
    elif isinstance(a, list):
        assert len(a) == len(b), where
        for i, (x, y) in enumerate(zip(a, b)):
            same_state(x, y, "%s[%d]" % (where, i))
    elif isinstance(a, np.ndarray):
        assert a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8)), where
    else:
        assert a == b, where


def same(got, want, what):
    if isinstance(got, list):
        assert len(got) == len(want), what
        for k, (g, w) in enumerate(zip(got, want)):
            same(g, w, "%s, model %d" % (what, k))
        return
    g, w = host(got), host(want)
    assert g.shape == w.shape and np.array_equal(g.view(np.uint8), w.view(np.uint8)), what


def same_everything(a, b, what, history=0):
    import torch
    torch.cuda.synchronize()
    same_state(a.state_dict(), b.state_dict(), what)
    if history:
        ids = np.arange(a.n_streams)
        same(a.audio_history(ids, history), b.audio_history(ids, history), what + ": audio history")


@pytest.mark.parametrize("blob", [F32, I8], ids=["f32", "int8"])
def test_every_path_against_the_int16_twin(torch_cuda, blob, monkeypatch):
    rng = np.random.default_rng(1)
    rates, fmts, n16 = RATES16, FMTS16, 48000                   # 3 s calls
    x, y = call(rng, rates, fmts, 0, n16)
    a, b = engines(StreamEngine, None, rates, fmts)
    same(a.features(dev(x), samples16=n16, mixed=True), b.features(dev(y), samples16=n16), "features")
    same_everything(a, b, "features")
    for path in ("device", "pageable", "pinned", "write-combined", "remote"):
        a, b = engines(StreamEngine, blob, rates, fmts, history=8192)
        for k in range(2):
            x, y = call(rng, rates, fmts, k * n16, n16)
            if path == "device":
                got, want = a.predict_clip(dev(x), samples16=n16, mixed=True), b.predict_clip(dev(y), samples16=n16)
            elif path == "pageable":
                got, want = a.predict_clip_host(x, samples16=n16, mixed=True), b.predict_clip_host(y, samples16=n16)
            elif path == "remote":
                buf = a.host_buffer(x.shape, np.uint8)
                buf[:] = x
                got = a.predict_clip_remote(buf.ctypes.data, x.shape[1], samples16=n16, tiles=3, mixed=True)
                want = b.predict_clip(dev(y), samples16=n16)
            else:
                buf = a.host_buffer(x.shape, np.uint8, write_combined=path == "write-combined")
                buf[:] = x
                got, want = a.predict_clip_host(buf, samples16=n16, mixed=True), b.predict_clip_host(y, samples16=n16)
            same(got, want, "%s call %d" % (path, k))
        same_everything(a, b, path, 8192)


def test_small_tiles_and_several_models_with_stream_sets(torch_cuda, monkeypatch):
    monkeypatch.setenv("MWW_SCRATCH_MB", "1")                   # a 3 s call then takes several tiles
    monkeypatch.setenv("MWW_MIN_TILE_STREAMS", "1")
    rng = np.random.default_rng(2)
    rates, fmts = np.tile(RATES16, 3), np.tile(FMTS16, 3)
    streams = [None, np.arange(0, rates.size, 3)]
    a, b = engines(MultiModelEngine, [F32, I8], rates, fmts, history=4096, streams=streams)
    t = 0
    for n16 in (48000, 480, 480, 32000):
        x, y = call(rng, rates, fmts, t, n16)
        same(a.predict_clip(dev(x), samples16=n16, mixed=True), b.predict_clip(dev(y), samples16=n16), "device %d" % n16)
        t += n16
        x, y = call(rng, rates, fmts, t, n16)
        same(a.predict_clip_host(x, samples16=n16, mixed=True), b.predict_clip_host(y, samples16=n16), "host %d" % n16)
        t += n16
    same_everything(a, b, "multi", 4096)


def test_live_calls_with_format_changes(torch_cuda):
    rng = np.random.default_rng(3)
    rates, fmts = RATES16, FMTS16.copy()
    for blob in (F32, I8):
        a, b = engines(StreamEngine, blob, rates, fmts, history=2048)
        for k in range(12):
            if k % 3 == 2:                                      # a caller switches some streams' formats between calls
                ids = rng.choice(rates.size, 5, replace=False)
                fmts[ids] = rng.integers(0, 4, ids.size)
                a.set_stream_formats(ids, fmts[ids])
                assert np.array_equal(a.stream_formats, fmts)
            x, y = call(rng, rates, fmts, 480 * k, 480)
            same(a.step(dev(x), mixed=True), b.step(dev(y)), "live call %d" % k)
        same_everything(a, b, "live", 2048)


def test_uniform_mixed_calls_equal_the_uniform_entry_points(torch_cuda):
    rng = np.random.default_rng(4)
    for fmt, law in ((ULAW, "ulaw"), (ALAW, "alaw"), (F32F, None), (S16, None)):
        rates = np.array([8000, 8000, 22050, 48000, 16000, 44100], np.int32)
        fmts = np.full(rates.size, fmt, np.int32)
        a, b = engines(StreamEngine, I8, rates, fmts)
        t = 0
        for n16 in (9600, 480, 480):
            x, _ = call(rng, rates, fmts, t, n16)
            dtype = {ULAW: np.uint8, ALAW: np.uint8, F32F: np.float32, S16: np.int16}[fmt]
            typed = np.ascontiguousarray(x).view(dtype)         # the same bytes as the format's own dtype
            same(a.predict_clip(dev(x), samples16=n16, mixed=True), b.predict_clip(dev(typed), samples16=n16, law=law), (fmt, n16))
            t += n16
        same_everything(a, b, "uniform %d" % fmt)


def test_padding_past_each_row_is_never_read(torch_cuda):
    rates, fmts = RATES16, FMTS16
    a = StreamEngine(F32, rates.size, 0, stream_rates=rates, stream_formats=fmts)
    b = StreamEngine(F32, rates.size, 0, stream_rates=rates, stream_formats=fmts)
    t = 0
    for k, n16 in enumerate((480, 9600, 480)):
        x0, _ = call(np.random.default_rng(k), rates, fmts, t, n16, pad=0x00)
        x1, _ = call(np.random.default_rng(k), rates, fmts, t, n16, pad=0xFF)
        wide = np.full((x1.shape[0], x1.shape[1] + 64), 0xFF, np.uint8)      # a wider pitch, NaN and full-scale bytes past each row
        wide[:, :x1.shape[1]] = x1
        same(a.predict_clip(dev(x0), samples16=n16, mixed=True), b.predict_clip(dev(wide), samples16=n16, mixed=True), "call %d" % k)
        t += n16
    same_everything(a, b, "padding")


def test_65536_streams_live(torch_cuda):
    S = 65536
    rng = np.random.default_rng(5)
    rates = np.array([8000, 8000, 48000, 16000], np.int32)[np.arange(S) % 4]
    fmts = np.array([ULAW, ALAW, F32F, S16], np.int32)[np.arange(S) % 4]
    rates[::7], fmts[::11] = 22050, F32F
    a, b = engines(StreamEngine, I8, rates, fmts)
    for k in range(3):
        x, y = call(rng, rates, fmts, 480 * k, 480)
        same(a.step(dev(x), mixed=True), b.step(dev(y)), "live call %d" % k)
    x, y = call(rng, rates, fmts, 1440, 4800)
    same(a.predict_clip_host(x, samples16=4800, mixed=True), b.predict_clip_host(y, samples16=4800), "host")
    same_everything(a, b, "65536")


def test_moved_streams_keep_their_formats(torch_cuda, tmp_path):
    rng = np.random.default_rng(6)
    rates, fmts = RATES16, FMTS16
    src, twin = engines(StreamEngine, F32, rates, fmts, history=4096)
    t = 0
    for n16 in (9600, 480):
        x, y = call(rng, rates, fmts, t, n16)
        src.predict_clip(dev(x), samples16=n16, mixed=True)
        twin.predict_clip(dev(y), samples16=n16)
        t += n16
    ids = np.array([0, 2, 5, 9, 12], np.int32)
    recs = src.export_streams(ids, history=4096, resampler=True)
    assert np.array_equal(recs.formats, fmts[ids])
    recs.save(tmp_path / "recs.npz")
    loaded = StreamRecords.load(tmp_path / "recs.npz", "cuda")
    assert np.array_equal(loaded.formats, fmts[ids])
    # the destination: the same counter, the streams at their rates; import gives them their formats
    dst = StreamEngine(F32, rates.size, 0, stream_rates=rates)
    dst.set_audio_history(4096)
    for n16 in (9600, 480):
        dst.predict_clip(dev(np.zeros((rates.size, int(inputs_for_rates(rates, 0, 10080).max())), np.int16)), samples16=n16)
    dst.import_streams(ids, loaded)
    assert np.array_equal(dst.stream_formats[ids], fmts[ids])
    for k in range(3):
        x, y = call(rng, rates, fmts, t, 480)
        x = x.copy()
        x[np.setdiff1d(np.arange(rates.size), ids)] = 0
        got, want = host(dst.step(dev(x), mixed=True)), host(twin.step(dev(y)))
        assert np.array_equal(got[ids].view(np.uint8), want[ids].view(np.uint8)), k
        t += 480
    import torch
    torch.cuda.synchronize()
    d, w = dst.state_dict(), twin.state_dict()
    for k in ("carry", "estimate", "nn", "pending", "resampler_history"):
        assert np.array_equal(d[k][ids].view(np.uint8), w[k][ids].view(np.uint8)), k
    same(dst.audio_history(ids, 4096), twin.audio_history(ids, 4096), "moved history")


def test_refusals_leave_the_handle_unchanged(torch_cuda):
    import torch
    rng = np.random.default_rng(7)
    rates, fmts = RATES16, FMTS16
    e, twin = engines(StreamEngine, F32, rates, fmts, history=2048)
    x, y = call(rng, rates, fmts, 0, 4800)
    e.predict_clip(dev(x), samples16=4800, mixed=True)
    twin.predict_clip(dev(y), samples16=4800)
    torch.cuda.synchronize()
    before = e.state_dict()
    L, h, st = e._L, e._h, e._cu_stream()
    x, y = call(rng, rates, fmts, 4800, 480)
    W = x.shape[1]
    big = torch.zeros((rates.size * (W + 8) + 8,), dtype=torch.uint8, device="cuda")
    hbig = np.zeros(rates.size * (W + 8) + 8, np.uint8)
    probs = torch.empty((rates.size, 8), dtype=torch.float32, device="cuda")
    probs_h = np.empty((rates.size, 8), np.float32)
    feat = torch.empty((rates.size, 8, 40), dtype=torch.uint16, device="cuda")
    ptrs, ptrs_h = (ctypes.c_void_p * 1)(probs.data_ptr()), (ctypes.c_void_p * 1)(probs_h.ctypes.data)
    maxp, got = (ctypes.c_int * 1)(8), ctypes.c_int(0)
    for base, stride, n16 in ((0, W - 4, 480), (0, W + 2, 480), (1, W, 480), (2, W + 4, 480), (0, W, 481), (0, W, -2)):
        d, hp = big.data_ptr() + base, hbig.ctypes.data + base
        calls = [
            L.mww_features_mixed(h, d, n16, stride, feat.data_ptr(), 8, ctypes.byref(got), st),
            L.mww_predict_clip_mixed(h, d, n16, stride, probs.data_ptr(), 8, ctypes.byref(got), st),
            L.mww_predict_clip_multi_mixed(h, d, n16, stride, ptrs, maxp, None, st),
            L.mww_predict_clip_host_mixed(h, hp, n16, stride, probs_h.ctypes.data, 8, ctypes.byref(got)),
            L.mww_predict_clip_host_multi_mixed(h, hp, n16, stride, ptrs_h, maxp, None),
            L.mww_predict_clip_remote_mixed(h, hp, n16, stride, probs.data_ptr(), 8, ctypes.byref(got), 4, st),
            L.mww_predict_clip_remote_multi_mixed(h, hp, n16, stride, ptrs, maxp, None, 0, st),
        ]
        assert calls == [-1] * 7, (base, stride, n16, calls)
    ids = np.array([1, 2], np.int32)
    for bad in (np.array([4, 0], np.int32), np.array([-1, 0], np.int32)):
        assert L.mww_set_stream_formats(h, ids.ctypes.data, bad.ctypes.data, 2, st) == -1
    dup = np.array([3, 3], np.int32)
    assert L.mww_set_stream_formats(h, dup.ctypes.data, np.zeros(2, np.int32).ctypes.data, 2, st) == -1
    with pytest.raises(ValueError):
        e.set_stream_formats([1], ["pcmu"])
    with pytest.raises(ValueError):
        e.step(dev(x), mixed=True, law="ulaw")
    torch.cuda.synchronize()
    same_state(e.state_dict(), before)
    assert np.array_equal(e.stream_formats, fmts)
    same(e.step(dev(x), mixed=True), twin.step(dev(y)), "after refusals")
    same_everything(e, twin, "after refusals", 2048)
    # a handle without per-stream rates: MWW_EUNSUPPORTED, nothing changed
    single = StreamEngine(F32, 4, 0, input_rate=48000)
    z = torch.zeros((4, 5760), dtype=torch.uint8, device="cuda")
    single.predict_clip(torch.zeros((4, 1440), dtype=torch.int16, device="cuda"))
    torch.cuda.synchronize()
    before = single.state_dict()
    assert single._L.mww_predict_clip_mixed(single._h, z.data_ptr(), 480, 5760, probs.data_ptr(), 8, ctypes.byref(got), st) == -5
    assert single._L.mww_set_stream_formats(single._h, ids.ctypes.data, np.array([1, 1], np.int32).ctypes.data, 2, st) == -5
    with pytest.raises(_lib.MwwError):
        single.set_stream_formats([0], "ulaw")
    with pytest.raises(ValueError):
        single.predict_clip(z, samples16=480, mixed=True)
    torch.cuda.synchronize()
    same_state(single.state_dict(), before)
    assert np.array_equal(single.stream_formats, np.zeros(4, np.int32))
