"""Each model of a multi-model handle on its own streams (mww_create_multi_streams), run with -m gpu on an H100.

The reference is an all-streams MultiModelEngine of the same containers given the same calls: for every member stream,
model k's probabilities and state rows must be bit-identical to the reference's rows of that stream.  Models: fp32
okay_nabu (wgmma clip and live kernels), int8 okay_nabu, the hybrid okay_nabu and the int8 run-time geometry of stride 17
(tests/generic_range.py's long_stride): the three fresh-state fills (zero, int8 zero points, run-time-geometry int8) and
every NN kernel family.  6 x SMs + 37 streams: past the live kernels' first persistent wave."""

import ctypes

import numpy as np
import pytest

from generic_range import GEOMETRIES, models as range_models
from microwakeword_b200 import _lib
from microwakeword_b200 import model_file as MF
from test_gpu_multi_model import _audio, _blobs as _multi_blobs

pytestmark = pytest.mark.gpu


def _blobs():
    f32, i8, hybrid, _, _ = _multi_blobs()
    _, ls8 = range_models(GEOMETRIES["long_stride"])
    return [f32, i8, hybrid, MF.write_container(ls8)]


def _S(torch):
    return 6 * torch.cuda.get_device_properties(0).multi_processor_count + 37


def _sets(S, which, seed=0):
    rng = np.random.default_rng(seed)
    kinds = {
        "all": None,
        "block": np.arange(S // 3, S // 3 + S // 4, dtype=np.int32),
        "interleaved": np.arange(1, S, 3, dtype=np.int32),
        "random": np.flatnonzero(rng.random(S) < 0.45).astype(np.int32),
        "empty": np.zeros(0, np.int32),
        "last": np.array([S - 1], np.int32),
    }
    return [kinds[w] for w in which]


MEMBERSHIPS = [("all", "block", "interleaved", "random"), ("interleaved", "random", "empty", "last"),
               ("random", "last", "all", "block"), ("empty", "interleaved", "block", "random")]


def _np(x):
    return x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)


class SubPair:
    """A MultiModelEngine with stream sets and an all-streams one of the same containers, fed the same calls."""

    def __init__(self, S, streams, blobs=None):
        from microwakeword_b200.engine import MultiModelEngine
        self.blobs = blobs or _blobs()
        self.ref = MultiModelEngine(self.blobs, S)
        self.sub = MultiModelEngine(self.blobs, S, streams=streams)
        self.S = S
        for k, s in enumerate(streams):
            assert np.array_equal(self.sub.streams[k], np.arange(S) if s is None else s)

    def all(self):
        return [self.ref, self.sub]

    def call(self, name, *args, **kw):
        want = getattr(self.ref, name)(*args, **kw)
        got = getattr(self.sub, name)(*args, **kw)
        for k, (g, w) in enumerate(zip(got, want)):
            g, w = _np(g), _np(w)
            ids = self.sub.streams[k]
            assert g.shape == (ids.size, w.shape[1]), (name, k, g.shape, w.shape)
            assert np.array_equal(g.view(np.int32), w[ids].view(np.int32)), (name, k)
        return got

    def check_state(self):
        d, r = self.sub.state_dict(), self.ref.state_dict()
        for key in ("carry", "estimate", "frontend_buffered"):
            assert np.array_equal(d[key], r[key]), key
        for k, (m, w) in enumerate(zip(d["models"], r["models"])):
            ids = self.sub.streams[k]
            assert np.array_equal(m["streams"], ids)
            assert m["pending_rows"] == w["pending_rows"], k
            assert np.array_equal(m["nn"], w["nn"][ids]), k
            assert np.array_equal(m["pending"], w["pending"][ids]), k
            info = _lib.MwwInfo()
            assert self.sub._L.mww_get_model_info(self.sub._h, k, ctypes.byref(info)) == 0 and info.n_streams == ids.size


@pytest.mark.parametrize("which", range(len(MEMBERSHIPS)))
def test_memberships_clip_and_live(torch_cuda, which):
    torch = torch_cuda
    S = _S(torch)
    p = SubPair(S, _sets(S, MEMBERSHIPS[which], which))
    for i, n in enumerate((48000, 47999)):
        p.call("predict_clip", _audio(torch, S, n, 100 + i))
    for i in range(5):
        p.call("step", _audio(torch, S, 480, 110 + i))
    p.check_state()


@pytest.mark.parametrize("which", [0, 1])
def test_call_types_in_uneven_tiles(torch_cuda, monkeypatch, which):
    """MWW_SCRATCH_MB=1 (read at create): every call is cut into many tiles, so member ranges span several uneven tiles and
    some tiles hold no member of a model.  Device clips (int16, float32, unaligned int16), host clips, remote clips in
    tiles, live steps."""
    torch = torch_cuda
    monkeypatch.setenv("MWW_SCRATCH_MB", "1")
    monkeypatch.setenv("MWW_MIN_TILE_STREAMS", "64")
    S = _S(torch)
    p = SubPair(S, _sets(S, MEMBERSHIPS[which], 10 + which))
    p.call("predict_clip", _audio(torch, S, 48000, 200))
    p.call("predict_clip", _audio(torch, S, 47999, 201, torch.float32))
    base = torch.empty((S, 48001 + 1), dtype=torch.int16, device="cuda")
    base[:, 1:] = _audio(torch, S, 48001, 202)
    view = base[:, 1:]
    assert view.data_ptr() % 16 != 0
    p.call("predict_clip", view)
    for i, n in enumerate((48000, 47999)):
        p.call("predict_clip_host", _audio(torch, S, n, 210 + i).cpu().numpy())
    p.call("predict_clip_host", (_audio(torch, S, 4801, 212, torch.float32)).cpu().numpy())
    for i, n in enumerate((48000, 4801)):
        a = _audio(torch, S, n, 220 + i)
        torch.cuda.synchronize()
        p.call("predict_clip_remote", a.data_ptr(), n, tiles=5)
        torch.cuda.synchronize()
    for i in range(4):
        p.call("step", _audio(torch, S, 480, 230 + i))
    p.check_state()


def test_window_step_320(torch_cuda):
    torch = torch_cuda
    S = _S(torch)
    p = SubPair(S, _sets(S, MEMBERSHIPS[0], 3))
    for e in p.all():
        e.set_window_step(320)
    for i, n in enumerate((48000, 47999, 4801)):
        p.call("predict_clip", _audio(torch, S, n, 300 + i))
    p.check_state()


def _fresh_rows(ref, k, rows, blobs, S):
    """write fresh model-k state (from a newly created engine) into the reference's rows `rows` of model k"""
    from microwakeword_b200.engine import MultiModelEngine
    fresh = MultiModelEngine(blobs, S).state_dict()["models"][k]
    cur = ref.state_dict()["models"][k]
    nn, pend = cur["nn"].copy(), cur["pending"].copy()
    nn[rows], pend[rows] = fresh["nn"][rows], fresh["pending"][rows]
    _lib.check(ref._h, ref._L.mww_set_model_state(ref._h, k, nn.ctypes.data, pend.ctypes.data, int(cur["pending_rows"])))


def test_membership_change_with_rotated_rings_and_pending_rows(torch_cuda):
    torch = torch_cuda
    S = _S(torch)
    blobs = _blobs()
    p = SubPair(S, _sets(S, MEMBERSHIPS[0], 4), blobs)
    p.call("predict_clip", _audio(torch, S, 47999, 400))
    for i in range(4):
        p.call("step", _audio(torch, S, 480, 401 + i))          # rotated rings; the stride-17 model holds pending rows
    assert any(r > 0 for r in p.sub.pending_rows)
    rng = np.random.default_rng(5)
    for round_ in range(2):
        for k in range(4):
            old = p.sub.streams[k]
            new = np.flatnonzero(rng.random(S) < 0.5).astype(np.int32) if (k + round_) % 2 == 0 else np.arange(S // 5, S, 2, dtype=np.int32)
            joiners = np.setdiff1d(new, old)
            p.sub.set_streams(k, new)
            assert np.array_equal(p.sub.streams[k], new)
            _fresh_rows(p.ref, k, joiners, blobs, S)
        p.check_state()
        p.call("step", _audio(torch, S, 480, 420 + round_))
        p.call("predict_clip", _audio(torch, S, 4801, 430 + round_))
        p.call("step", _audio(torch, S, 480, 440 + round_))
        p.check_state()
    # back to all streams (None)
    joiners = np.setdiff1d(np.arange(S), p.sub.streams[3])
    p.sub.set_streams(3, None)
    _fresh_rows(p.ref, 3, joiners, blobs, S)
    p.call("step", _audio(torch, S, 480, 450))
    p.check_state()


def test_reset_by_host_and_device_ids(torch_cuda):
    torch = torch_cuda
    S = _S(torch)
    p = SubPair(S, _sets(S, MEMBERSHIPS[1], 6))
    p.call("predict_clip", _audio(torch, S, 48000, 500))
    p.call("step", _audio(torch, S, 480, 501))
    for e in p.all():
        e.reset(list(range(0, S, 7)) + [S - 1])
    p.call("step", _audio(torch, S, 480, 502))
    ids = torch.tensor([3, S - 1, 5, 1] + list(range(10, S, 4)) + [-2, S + 5], dtype=torch.int32, device="cuda")
    for e in p.all():
        e.reset(ids)
    p.check_state()
    p.call("step", _audio(torch, S, 480, 503))
    p.call("predict_clip", _audio(torch, S, 48000, 504))
    p.check_state()


def test_snapshot_into_a_fresh_engine_continues_exactly(torch_cuda):
    from microwakeword_b200.engine import MultiModelEngine
    torch = torch_cuda
    S = _S(torch)
    blobs = _blobs()
    sets = _sets(S, MEMBERSHIPS[3], 7)
    a = MultiModelEngine(blobs, S, streams=sets)
    a.predict_clip(_audio(torch, S, 47999, 600))
    for i in range(4):
        a.step(_audio(torch, S, 480, 601 + i))
    snap = a.state_dict()
    b = MultiModelEngine(blobs, S, streams=sets)
    c = MultiModelEngine(blobs, S)                                # restores the membership before the state
    b.load_state_dict(snap)
    c.load_state_dict(snap)
    for k in range(4):
        assert np.array_equal(c.streams[k], a.streams[k])
    for x in (_audio(torch, S, 48001, 610), _audio(torch, S, 480, 611)):
        ga, gb, gc = a.predict_clip(x), b.predict_clip(x), c.predict_clip(x)
        for k in range(4):
            assert torch.equal(ga[k].view(torch.int32), gb[k].view(torch.int32)), k
            assert torch.equal(ga[k].view(torch.int32), gc[k].view(torch.int32)), k


def test_refusals(torch_cuda):
    from microwakeword_b200.engine import MultiModelEngine
    torch = torch_cuda
    S = 70
    blobs = _blobs()
    # the one-model entry points refuse a K = 1 handle whose model is on a subset of the streams
    one = MultiModelEngine(blobs[:1], S, streams=[np.arange(0, S, 2, dtype=np.int32)])
    L, h, cs = one._L, one._h, one._cu_stream()
    a16 = _audio(torch, S, 480, 700)
    a32 = a16.to(torch.float32)
    probs = torch.empty((S, 64), device="cuda")
    got = ctypes.c_int(0)
    host = np.zeros((S, 480), np.int16)
    hprobs = np.zeros((S, 64), np.float32)
    nn = np.zeros((S, one.state_elements[0]), np.float32)
    pend_buf = np.zeros((S, 2, 40), np.float32)
    calls = {
        "mww_predict_clip": lambda: L.mww_predict_clip(h, a16.data_ptr(), 480, 480, probs.data_ptr(), 64, ctypes.byref(got), cs),
        "mww_predict_clip_f32": lambda: L.mww_predict_clip_f32(h, a32.data_ptr(), 480, 480, probs.data_ptr(), 64, ctypes.byref(got), cs),
        "mww_predict_clip_host": lambda: L.mww_predict_clip_host(h, host.ctypes.data, 480, 480, hprobs.ctypes.data, 64, ctypes.byref(got)),
        "mww_predict_clip_host_f32": lambda: L.mww_predict_clip_host_f32(h, host.ctypes.data, 0, 0, hprobs.ctypes.data, 64, ctypes.byref(got)),
        "mww_predict_clip_remote": lambda: L.mww_predict_clip_remote(h, a16.data_ptr(), 480, 480, probs.data_ptr(), 64, ctypes.byref(got), 2, cs),
        "mww_infer_features": lambda: L.mww_infer_features(h, probs.data_ptr(), 1, 3, 3, probs.data_ptr(), 64, ctypes.byref(got), cs),
        "mww_copy_nn_state": lambda: L.mww_copy_nn_state(h, (ctypes.c_int32 * 1)(0), h, (ctypes.c_int32 * 1)(1), 1, cs),
        "mww_get_state": lambda: L.mww_get_state(h, None, None, nn.ctypes.data, None),
        "mww_set_state": lambda: L.mww_set_state(h, None, 0, None, nn.ctypes.data, pend_buf.ctypes.data, 0),
    }
    launches, buffered = one.launch_count, one.frontend_buffered
    for name, fn in calls.items():
        assert fn() == -1, name
        msg = L.mww_last_error(h).decode()
        assert name in msg and "subset of the streams" in msg, (name, msg)
    assert (one.launch_count, one.frontend_buffered) == (launches, buffered)

    # output buffers: one row per member; a too-small one is refused before any launch
    m = MultiModelEngine(blobs, S, streams=[None, np.arange(5, 40, dtype=np.int32), np.zeros(0, np.int32), np.array([S - 1], np.int32)])
    x = _audio(torch, S, 48000, 701)
    steps = m._steps(48000)
    with pytest.raises(ValueError):
        m.predict_clip(x, out=[torch.empty((S, s), device="cuda") for s in steps])
    out = [torch.empty((n.size, s), device="cuda") for n, s in zip(m.streams, steps)]
    out[1] = torch.empty((35, steps[1] - 1), device="cuda")
    launches = m.launch_count
    with pytest.raises(_lib.MwwError) as e:
        m.predict_clip(x, out=out)
    assert e.value.code == -1 and "model 1" in str(e.value) and m.launch_count == launches

    # a model without members takes a NULL buffer and still reports its steps
    ptrs = (ctypes.c_void_p * 4)(*[None if k == 2 else out[k].data_ptr() for k in range(4)])
    maxp = (ctypes.c_int * 4)(*[0 if k == 2 else steps[k] for k in range(4)])
    outs = (ctypes.c_int * 4)()
    out[1] = torch.empty((35, steps[1]), device="cuda")
    ptrs[1] = out[1].data_ptr()
    assert L.mww_predict_clip_multi(m._h, x.data_ptr(), 48000, 48000, ptrs, maxp, outs, m._cu_stream()) == 0
    assert list(outs) == steps and steps[2] > 0

    # bad ids in mww_set_model_streams: refused, the handle continues unchanged (against a twin given the same calls)
    twin = MultiModelEngine(blobs, S, streams=[None, np.arange(5, 40, dtype=np.int32), np.zeros(0, np.int32), np.array([S - 1], np.int32)])
    twin.predict_clip(x)
    for ids in ([3, 2], [1, 1], [-1, 4], [0, S]):
        a = np.asarray(ids, np.int32)
        assert m._L.mww_set_model_streams(m._h, 1, a.ctypes.data, a.size, m._cu_stream()) == -1
        assert "strictly increasing" in m._L.mww_last_error(m._h).decode()
    a = np.arange(3, dtype=np.int32)
    assert m._L.mww_set_model_streams(m._h, 1, a.ctypes.data, -1, m._cu_stream()) == -1
    assert m._L.mww_set_model_streams(m._h, 4, a.ctypes.data, 3, m._cu_stream()) == -1
    with pytest.raises(ValueError):
        m.set_streams(1, [5, 4])
    assert np.array_equal(m.streams[1], np.arange(5, 40))
    y = _audio(torch, S, 480, 702)
    for g, w in zip(m.predict_clip(y), twin.predict_clip(y)):
        assert torch.equal(g.view(torch.int32), w.view(torch.int32))


def test_launch_counts(torch_cuda):
    """All streams and one contiguous block issue the launches of a handle without stream sets; an interleaved set adds
    one row gather per model per tile (one tile at the default scratch budget)."""
    from microwakeword_b200.engine import MultiModelEngine
    torch = torch_cuda
    S = _S(torch)
    blobs = _blobs()
    block = np.arange(S // 4, S // 2, dtype=np.int32)
    inter = np.arange(0, S, 2, dtype=np.int32)
    base = MultiModelEngine(blobs, S)
    same = MultiModelEngine(blobs, S, streams=[None, block, np.arange(S, dtype=np.int32), block])
    gath = MultiModelEngine(blobs, S, streams=[inter, None, inter, block])
    for n in (48000, 480, 480, 47999):
        x = _audio(torch, S, n, 800 + n)
        before = [e.launch_count for e in (base, same, gath)]
        for e in (base, same, gath):
            e.predict_clip(x)
        d = [e.launch_count - b for e, b in zip((base, same, gath), before)]
        assert d[1] == d[0], (n, d)
        assert d[2] == d[0] + 2, (n, d)
