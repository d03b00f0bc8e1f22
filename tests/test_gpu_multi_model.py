"""Several models over one frontend (mww_create_multi / MultiModelEngine), run with -m gpu on an H100.

For every model k the probabilities and NN state must be bit-identical to a separate StreamEngine of that model given the
same calls, and the shared frontend state bit-identical to any single engine's.  Models: fp32 okay_nabu (wgmma clip and
live kernels), int8 okay_nabu, the hybrid okay_nabu (generic hybrid kernel) and two run-time geometries of stride 17, fp32
and int8 (tests/generic_range.py's long_stride)."""

import ctypes
import functools
import os

import numpy as np
import pytest

import tflite_hybrid_writer as HW
from conftest import GOLDEN
from generic_range import GEOMETRIES, models as range_models
from microwakeword_b200 import _lib
from microwakeword_b200 import model_file as MF
from microwakeword_b200 import tflite_file as TF

pytestmark = pytest.mark.gpu


@functools.lru_cache(maxsize=None)
def _blobs():
    f32 = open(os.path.join(GOLDEN, "okay_nabu_synth_f32.mww"), "rb").read()
    i8 = open(os.path.join(GOLDEN, "okay_nabu_synth_int8.mww"), "rb").read()
    hybrid = MF.write_container(TF.tensors_from_tflite(HW.write_hybrid_mixednet(MF.load(os.path.join(GOLDEN, "okay_nabu_synth_f32.mww")),
                                                                                  lambda op, n: n >= 1024, True)))
    ls32, ls8 = range_models(GEOMETRIES["long_stride"])
    return (f32, i8, hybrid, MF.write_container(ls32), MF.write_container(ls8))


def _audio(torch, S, n, seed, dtype=None):
    """tones in noise; above 1 021 streams, stream s repeats stream s % 1 021 (a prime) to keep the generator's memory small"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    P = min(S, 1021)
    t = torch.arange(n, device="cuda", dtype=torch.float32)
    f = 200.0 + 1800.0 * torch.rand(P, 1, device="cuda", generator=g)
    x = 6000.0 * torch.sin(t[None, :] * f * (2 * np.pi / 16000)) + 1500.0 * torch.randn(P, n, device="cuda", generator=g)
    x = x.clamp(-32768, 32767).to(torch.int16)
    if S > P:
        x = x[torch.arange(S, device="cuda") % P]
    return x if dtype is None else (x.to(torch.float32) / 32768.0)


class Pair:
    """One MultiModelEngine and one StreamEngine per model, fed the same calls; every call's results are compared."""

    def __init__(self, S, blobs=None):
        from microwakeword_b200.engine import MultiModelEngine, StreamEngine
        self.blobs = blobs or _blobs()
        self.multi = MultiModelEngine(list(self.blobs), S)
        self.singles = [StreamEngine(b, S) for b in self.blobs]
        self.S = S

    def all(self):
        return [self.multi] + self.singles

    def call(self, name, *args, **kw):
        got = getattr(self.multi, name)(*args, **kw)
        want = [getattr(e, name)(*args, **kw) for e in self.singles]
        assert len(got) == len(want)
        for k, (g, w) in enumerate(zip(got, want)):
            g = g.cpu().numpy() if hasattr(g, "cpu") else np.asarray(g)
            w = w.cpu().numpy() if hasattr(w, "cpu") else np.asarray(w)
            assert g.shape == w.shape, (name, k, g.shape, w.shape)
            assert np.array_equal(g.view(np.int32), w.view(np.int32)), (name, k)
        return got

    def check_state(self):
        d = self.multi.state_dict()
        for k, e in enumerate(self.singles):
            s = e.state_dict()
            if k == 0:
                for key in ("carry", "estimate", "frontend_buffered"):
                    assert np.array_equal(d[key], s[key]), key
            m = d["models"][k]
            assert m["pending_rows"] == s["pending_rows"], k
            assert np.array_equal(m["nn"], s["nn"]), k
            assert np.array_equal(m["pending"], s["pending"]), k


def _sms(torch):
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("which", range(5))
def test_clip_calls_match_separate_engines(torch_cuda, which):
    """3 s clips, then 47 999 and 48 001 samples: the models enter later calls with different pending rows.  1 and 70
    streams; 12 x SMs - 1 (unfused K1 + K2); 6 x SMs + 37; 65 536 (fused clip frontend, wgmma)."""
    torch = torch_cuda
    sms = _sms(torch)
    S = [1, 70, 12 * sms - 1, 6 * sms + 37, 65536][which]
    p = Pair(S)
    for i, n in enumerate((48000, 47999, 48001)):
        got = p.call("predict_clip", _audio(torch, S, n, 10 + i))
        if i == 0:
            assert [g.shape[1] for g in got] == [99, 99, 99, 17, 17]          # 298 rows at strides 3 and 17
    p.check_state()


def test_live_steps_resets_and_clip(torch_cuda):
    """56 live 480-sample steps (each okay_nabu model's live kernel, rings rotating per model) with a reset by host ids and
    one by CUDA ids in the middle, then a clip call (rings canonicalised per model), then live steps again."""
    torch = torch_cuda
    S = 6 * _sms(torch) + 37
    p = Pair(S)
    audio = _audio(torch, S, 480 * 80 + 48000, 3)
    pos = 0
    for i in range(56):
        p.call("step", audio[:, pos:pos + 480].contiguous())
        pos += 480
        if i == 20:
            for e in p.all():
                e.reset(list(range(0, S, 7)))
        if i == 40:
            ids = torch.arange(3, S, 5, dtype=torch.int32, device="cuda")
            for e in p.all():
                e.reset(ids)
    p.check_state()
    p.call("predict_clip", audio[:, pos:pos + 48000].contiguous())
    pos += 48000
    for _ in range(24):
        p.call("step", audio[:, pos:pos + 480].contiguous())
        pos += 480
    p.check_state()


def test_float32_and_unaligned_int16_audio(torch_cuda):
    torch = torch_cuda
    S = 70
    p = Pair(S)
    p.call("predict_clip", _audio(torch, S, 48000, 5, torch.float32))
    base = torch.empty((S, 48001 + 1), dtype=torch.int16, device="cuda")
    base[:, 1:] = _audio(torch, S, 48001, 6)
    view = base[:, 1:]
    assert view.data_ptr() % 16 != 0 and view.stride(0) == 48002
    p.call("predict_clip", view)
    p.call("step", _audio(torch, S, 480, 7, torch.float32))
    p.check_state()


def test_window_step_320(torch_cuda):
    torch = torch_cuda
    S = 70
    p = Pair(S)
    for e in p.all():
        e.set_window_step(320)
    for i, n in enumerate((48000, 47999, 4801)):
        p.call("predict_clip", _audio(torch, S, n, 20 + i))
    p.check_state()


def test_stream_tiles_from_the_scratch_budget(torch_cuda, monkeypatch):
    """MWW_SCRATCH_MB=1 (read at create): every call is cut into many stream tiles, the frontend and the models of each tile
    at non-zero stream offsets"""
    torch = torch_cuda
    monkeypatch.setenv("MWW_SCRATCH_MB", "1")
    S = 6 * _sms(torch) + 37
    p = Pair(S)
    for i, n in enumerate((48000, 47999)):
        p.call("predict_clip", _audio(torch, S, n, 30 + i))
    p.call("step", _audio(torch, S, 480, 33))
    p.check_state()


def test_host_path_in_several_tiles_copies_each_tile_once(torch_cuda, monkeypatch):
    torch = torch_cuda
    monkeypatch.setenv("MWW_MIN_TILE_STREAMS", "64")
    S = 6 * _sms(torch) + 37
    p = Pair(S)
    for e in p.all():
        e.profile(True)
    for i, n in enumerate((48000, 47999, 48001)):
        a = _audio(torch, S, n, 40 + i).cpu().numpy()
        p.call("predict_clip_host", a)
    tiles = -(-S // max(-(-S // 16), 64))
    tl = p.multi.timeline_read()
    assert tl.shape[0] == tiles == p.singles[0].timeline_read().shape[0] > 1
    assert (np.diff(tl[:, 0]) > 0).all()                   # one copy per tile, in order
    p.check_state()


def test_remote_path_from_a_local_source_in_tiles(torch_cuda):
    torch = torch_cuda
    S = 6 * _sms(torch) + 37
    p = Pair(S)
    for i, n in enumerate((48000, 47999)):
        a = _audio(torch, S, n, 50 + i)
        torch.cuda.synchronize()
        p.call("predict_clip_remote", a.data_ptr(), n, tiles=5)
    torch.cuda.synchronize()
    p.check_state()


def test_snapshot_into_a_fresh_engine_continues_exactly(torch_cuda):
    from microwakeword_b200.engine import MultiModelEngine
    torch = torch_cuda
    S = 70
    blobs = list(_blobs())
    a = MultiModelEngine(blobs, S)
    first = _audio(torch, S, 47999, 60)
    live = [_audio(torch, S, 480, 61 + i) for i in range(5)]
    after = _audio(torch, S, 48001, 70)
    a.predict_clip(first)
    for x in live:
        a.step(x)                                           # rings left rotated: the snapshot canonicalises them
    snap = a.state_dict()
    assert len(set(m["pending_rows"] for m in snap["models"])) > 1
    b = MultiModelEngine(blobs, S)
    b.load_state_dict(snap)
    for x in (after, live[0]):
        ga, gb = a.predict_clip(x), b.predict_clip(x)
        for k in range(len(blobs)):
            assert torch.equal(ga[k].view(torch.int32), gb[k].view(torch.int32)), k
    da, db = a.state_dict(), b.state_dict()
    assert np.array_equal(da["carry"], db["carry"]) and np.array_equal(da["estimate"], db["estimate"])
    for ma, mb in zip(da["models"], db["models"]):
        assert np.array_equal(ma["nn"], mb["nn"]) and ma["pending_rows"] == mb["pending_rows"]


@pytest.mark.parametrize("n", [48000, 480])
def test_frontend_runs_once_whatever_k(torch_cuda, n):
    from microwakeword_b200.engine import MultiModelEngine, StreamEngine
    torch = torch_cuda
    S = 70
    blobs = list(_blobs())
    audio = _audio(torch, S, n, 80)
    one = StreamEngine(blobs[0], S)
    multi = MultiModelEngine(blobs, S)
    singles = [StreamEngine(b, S) for b in blobs]
    for e in [one, multi] + singles:
        e.profile(True)
        e.predict_clip(audio)
    want, got = one.profile_read(), multi.profile_read()
    for cls in ("k1_spectral", "k2_temporal", "carry_update"):
        assert got[cls][1] == want[cls][1], (cls, got, want)
    assert got["mixednet"][1] == sum(e.profile_read()["mixednet"][1] for e in singles)


def test_errors(torch_cuda):
    from microwakeword_b200.engine import MultiModelEngine, StreamEngine
    torch = torch_cuda
    S = 70
    f32, i8, hybrid, ls32, _ = _blobs()
    with pytest.raises(_lib.MwwError) as e:
        MultiModelEngine([], S)
    assert e.value.code == -1
    corrupt = b"MWWB200\0" + b"\x01\0\0\0\x05\0\0\0\xff\xff\0\0" + b"\0" * 64
    with pytest.raises(_lib.MwwError) as e:
        MultiModelEngine([f32, i8, corrupt, ls32], S)
    assert e.value.code == -2 and "model 2" in str(e.value)

    # a too-small buffer for one model: refused before any launch, no state change
    m = MultiModelEngine([f32, ls32], S)
    m.predict_clip(_audio(torch, S, 4000, 90))
    launches, buffered, pend = m.launch_count, m.frontend_buffered, m.pending_rows
    steps = m._steps(48000)
    out = [torch.empty((S, steps[0]), device="cuda"), torch.empty((S, steps[1] - 1), device="cuda")]
    with pytest.raises(_lib.MwwError) as e:
        m.predict_clip(_audio(torch, S, 48000, 91), out=out)
    assert e.value.code == -1 and "model 1" in str(e.value)
    assert (m.launch_count, m.frontend_buffered, m.pending_rows) == (launches, buffered, pend)

    # the one-model entry points refuse a K = 2 handle
    L, h = m._L, m._h
    a16 = _audio(torch, S, 480, 92)
    a32 = a16.to(torch.float32)
    probs = torch.empty((S, 64), device="cuda")
    got = ctypes.c_int(0)
    cs = m._cu_stream()
    host = np.zeros((S, 480), np.int16)
    hprobs = np.zeros((S, 64), np.float32)
    nn = np.zeros((S, m.state_elements[0]), np.float32)
    pend_buf = np.zeros((S, 2, 40), np.float32)
    carry, est = np.zeros((S, 480), np.int16), np.zeros((S, 40), np.uint32)
    calls = {
        "mww_predict_clip": lambda: L.mww_predict_clip(h, a16.data_ptr(), 480, 480, probs.data_ptr(), 64, ctypes.byref(got), cs),
        "mww_predict_clip_f32": lambda: L.mww_predict_clip_f32(h, a32.data_ptr(), 480, 480, probs.data_ptr(), 64, ctypes.byref(got), cs),
        "mww_predict_clip_host": lambda: L.mww_predict_clip_host(h, host.ctypes.data, 480, 480, hprobs.ctypes.data, 64, ctypes.byref(got)),
        "mww_predict_clip_remote": lambda: L.mww_predict_clip_remote(h, a16.data_ptr(), 480, 480, probs.data_ptr(), 64, ctypes.byref(got), 2, cs),
        "mww_infer_features": lambda: L.mww_infer_features(h, probs.data_ptr(), 1, 3, 3, probs.data_ptr(), 64, ctypes.byref(got), cs),
        "mww_copy_nn_state": lambda: L.mww_copy_nn_state(h, (ctypes.c_int32 * 1)(0), h, (ctypes.c_int32 * 1)(1), 1, cs),
        "mww_get_state": lambda: L.mww_get_state(h, None, None, nn.ctypes.data, None),
        "mww_set_state": lambda: L.mww_set_state(h, None, 0, None, nn.ctypes.data, pend_buf.ctypes.data, 0),
    }
    for name, fn in calls.items():
        assert fn() == -1, name
        msg = L.mww_last_error(h).decode()
        assert name in msg and "2 models" in msg, (name, msg)
    assert (m.launch_count, m.frontend_buffered, m.pending_rows) == (launches, buffered, pend)
    # without NN arrays the state calls move the shared frontend only
    assert L.mww_get_state(h, carry.ctypes.data, est.ctypes.data, None, None) == 0
    assert L.mww_set_state(h, carry.ctypes.data, buffered, est.ctypes.data, None, None, 0) == 0
    assert m.pending_rows == pend

    # a K = 1 multi handle behaves exactly like mww_create, one-model entry points included
    one, ref = MultiModelEngine([f32], S), StreamEngine(f32, S)
    for n in (47999, 480, 48001):
        x = _audio(torch, S, n, 93 + n)
        g, w = one.predict_clip(x)[0], ref.predict_clip(x)
        assert torch.equal(g.view(torch.int32), w.view(torch.int32))
    assert one.launch_count == ref.launch_count
    x = _audio(torch, S, 480, 99)
    w = ref.predict_clip(x)
    assert L.mww_predict_clip(one._h, x.data_ptr(), 480, 480, probs.data_ptr(), 64, ctypes.byref(got), one._cu_stream()) == 0
    assert torch.equal(probs[:, :got.value].view(torch.int32), w.view(torch.int32))
    s1, s2 = one.state_dict(), ref.state_dict()
    assert np.array_equal(s1["carry"], s2["carry"]) and np.array_equal(s1["estimate"], s2["estimate"])
    assert np.array_equal(s1["models"][0]["nn"], s2["nn"]) and np.array_equal(s1["models"][0]["pending"], s2["pending"])
