"""Moving streams between handles as packed records (mww_export_streams / mww_import_streams), run with -m gpu on an H100.

The central property needs no oracle: a stream that moves continues bit for bit as if it had stayed, and every stream that
did not move continues as in a twin handle that never imported anything.  Models: fp32, int8 and hybrid okay_nabu and the
run-time geometry of stride 17 (tests/generic_range.py's long_stride), fp32 and int8.  6 x SMs + 37 streams: past the live
kernels' first persistent wave.  Every refusal here is a checked argument error returned before any device work."""

import numpy as np
import pytest

from microwakeword_b200 import _lib
from test_gpu_multi_model import _audio, _blobs

pytestmark = pytest.mark.gpu

KINDS = ("f32", "int8", "hybrid", "generic_f32", "generic_int8")
FRONTEND_BYTES = 16 + 960 + 160


def _blob(kind):
    return dict(zip(KINDS, _blobs()))[kind]


def _S(torch):
    return 6 * torch.cuda.get_device_properties(0).multi_processor_count + 37


def _np(x):
    return x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)


def _bits(x):
    return _np(x).view(np.int32)


def _idx(torch, ids):
    return torch.from_numpy(np.asarray(ids, np.int64)).cuda()


def _serve(torch, eng, n_live, seed, clip=4801):
    """a clip call that leaves pending rows and a partial window (321 samples), then live calls that rotate the rings"""
    S = eng.n_streams
    eng.predict_clip(_audio(torch, S, clip, seed))
    for i in range(n_live):
        eng.step(_audio(torch, S, 480, seed + 1 + i))


def _routed(torch, a_audio, S_B, seed, src, dst):
    """audio for the destination handle: its own, with stream dst[i] hearing what stream src[i] of the source hears"""
    b = _audio(torch, S_B, a_audio.shape[1], seed)
    b[_idx(torch, dst)] = a_audio[_idx(torch, src)]
    return b


def _pad16(n):
    return (n + 15) // 16 * 16


def _decode(rec, engines_state):
    """records [n, record_bytes] uint8 -> (mask, carry, estimate, [(nn, pending) per model]) by the documented layout;
    engines_state: [(dtype, state_elements, pending rows kept)] per model"""
    mask = rec[:, :8].copy().view(np.uint64).ravel()
    carry = rec[:, 16:976].copy().view(np.int16)
    est = rec[:, 976:1136].copy().view(np.uint32)
    off, models = FRONTEND_BYTES, []
    for dt, elems, cap in engines_state:
        es = np.dtype(dt).itemsize
        nn = rec[:, off:off + elems * es].copy().view(dt)
        assert not rec[:, off + elems * es:off + _pad16(elems * es)].any()
        off += _pad16(elems * es)
        pend = rec[:, off:off + cap * 40 * es].copy().view(dt).reshape(-1, cap, 40)
        assert not rec[:, off + cap * 40 * es:off + _pad16(cap * 40 * es)].any()
        off += _pad16(cap * 40 * es)
        models.append((nn, pend))
    assert off == rec.shape[1]
    return mask, carry, est, models


# ---- continuation ---------------------------------------------------------------------------------------------------------
# (kind, live calls the destination made before the import; the source made 7).  The state always moves exactly.  What a
# moved stream computes next is bit-identical wherever the arithmetic does not depend on the ring rotation: every integer
# model, the hybrid and run-time-geometry kernels (canonical rings), and fp32 okay_nabu at the rotation it left.  The fp32
# live-step kernel adds a ring's taps in physical row order, so at another rotation the same state gives sums that differ
# in the last bits -- as they do for a stream that stays, between two handles with different live-call histories.
CASES = [("f32", 7), ("f32", 12), ("int8", 12), ("hybrid", 12), ("generic_f32", 7), ("generic_int8", 7)]


@pytest.mark.parametrize("kind,dst_live", CASES)
def test_moved_streams_continue_as_if_they_had_stayed(torch_cuda, kind, dst_live):
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    exact = not (kind == "f32" and dst_live != 7)
    SA = _S(torch)
    SB = SA + 91
    A, B, twin = (StreamEngine(_blob(kind), S) for S in (SA, SB, SB))
    _serve(torch, A, 7, 10)
    for e in (B, twin):
        _serve(torch, e, dst_live, 50)                 # same counters, other audio
    rng = np.random.default_rng(3)
    src, dst = rng.permutation(SA)[:200].astype(np.int32), rng.permutation(SB)[:200].astype(np.int32)
    others = np.setdiff1d(np.arange(SB), dst)
    before = B.launch_count
    B.import_streams(dst, A.export_streams(torch.from_numpy(src)))
    assert B.launch_count - before <= 3                # frontend, model, int8 fresh fill: whatever the number of streams
    steps = 0
    for i, n in enumerate((480, 480, 480, 4799, 480, 480)):
        a = _audio(torch, SA, n, 100 + i)
        b = _routed(torch, a, SB, 200 + i, src, dst)
        pa, pb, pt = A.predict_clip(a), B.predict_clip(b), twin.predict_clip(b)
        assert pa.shape[1] == pb.shape[1] == pt.shape[1]
        if exact:
            assert np.array_equal(_bits(pb)[dst], _bits(pa)[src]), (kind, i)
        else:
            assert np.abs(_np(pb)[dst] - _np(pa)[src]).max() <= 1e-6, (kind, i)
        assert np.array_equal(_bits(pb)[others], _bits(pt)[others]), (kind, i)
        steps += pa.shape[1]
    assert steps >= 3
    sa, sb, st = A.state_dict(), B.state_dict(), twin.state_dict()
    for key in ("carry", "estimate", "nn", "pending"):
        if exact or key != "nn":
            assert np.array_equal(sb[key][dst], sa[key][src]), (kind, key)
        else:
            assert np.allclose(sb[key][dst], sa[key][src], rtol=0, atol=1e-4), (kind, key)
        assert np.array_equal(sb[key][others], st[key][others]), (kind, key)
    assert sa["frontend_buffered"] == sb["frontend_buffered"] and sa["pending_rows"] == sb["pending_rows"]


@pytest.mark.parametrize("kind", ["f32", "int8"])
def test_state_arrives_exactly_at_another_rotation(torch_cuda, kind):
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    SA = _S(torch)
    SB = SA + 91
    A, B, twin = (StreamEngine(_blob(kind), S) for S in (SA, SB, SB))
    _serve(torch, A, 7, 10)
    for e in (B, twin):
        _serve(torch, e, 12, 50)
    rng = np.random.default_rng(8)
    src, dst = rng.permutation(SA)[:200].astype(np.int32), rng.permutation(SB)[:200].astype(np.int32)
    others = np.setdiff1d(np.arange(SB), dst)
    B.import_streams(dst, A.export_streams(src))
    sa, sb, st = A.state_dict(), B.state_dict(), twin.state_dict()
    for key in ("carry", "estimate", "nn", "pending"):
        assert np.array_equal(sb[key][dst], sa[key][src]), (kind, key)
        assert np.array_equal(sb[key][others], st[key][others]), (kind, key)


# ---- record format; export leaves the handle alone ----------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["f32", "int8", "generic_int8"])
def test_records_hold_the_documented_fields_and_export_changes_nothing(torch_cuda, kind):
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    S = _S(torch)
    A, twin = StreamEngine(_blob(kind), S), StreamEngine(_blob(kind), S)
    for e in (A, twin):
        _serve(torch, e, 7, 20)
    ids = np.random.default_rng(1).permutation(S)[:150].astype(np.int32)
    ids[7] = ids[3]                                    # export allows an id twice
    c0 = A.launch_count
    A.export_streams(ids)
    assert A.launch_count - c0 == 2                    # the frontend parts and the model: nothing canonicalised
    c0, t0 = A.launch_count, twin.launch_count
    a = _audio(torch, S, 480, 40)
    assert np.array_equal(_bits(A.step(a)), _bits(twin.step(a)))
    assert A.launch_count - c0 == twin.launch_count - t0
    rec = A.export_streams(ids)
    torch.cuda.synchronize()
    d = A.state_dict()                                 # canonical rings, read after the export
    dt = np.int8 if A.is_quantized else np.float32
    mask, carry, est, models = _decode(rec.data.cpu().numpy(), [(dt, A.state_elements, max(A.stride - 1, 1))])
    assert (mask == 1).all()
    assert np.array_equal(carry, d["carry"][ids]) and np.array_equal(est, d["estimate"][ids])
    assert np.array_equal(models[0][0], d["nn"][ids]) and np.array_equal(models[0][1], d["pending"][ids])
    L = rec.layout
    assert (L.record_bytes, L.n_models, L.frontend_buffered, L.hop_samples) == (rec.data.shape[1], 1, d["frontend_buffered"], 160)
    assert L.pending_rows[0] == d["pending_rows"] and L.rows_are_features[0] == 1
    own = A.stream_layout()
    assert bytes(own) == bytes(L)


def test_frontend_only_handles(torch_cuda):
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    A, B = StreamEngine(None, 300), StreamEngine(None, 200)
    A.features(_audio(torch, 300, 4801, 1))
    B.features(_audio(torch, 200, 4801, 2))
    src, dst = np.asarray([299, 0, 17], np.int32), np.asarray([5, 199, 0], np.int32)
    rec = A.export_streams(src)
    assert rec.data.shape == (3, FRONTEND_BYTES) and rec.layout.n_models == 0
    B.import_streams(dst, rec)
    a = _audio(torch, 300, 1600, 3)
    fa, fb = A.features(a), B.features(_routed(torch, a, 200, 4, src, dst))
    assert np.array_equal(_np(fb.view(torch.int16))[dst], _np(fa.view(torch.int16))[src])


# ---- several models on their own stream sets --------------------------------------------------------------------------------
def test_stream_sets_membership_rule(torch_cuda):
    """Reference R: an all-streams engine given the source's calls, in which model k restarts (leaves and rejoins the set)
    exactly the moved streams the source held no model-k state for.  Every destination member then equals R's source stream."""
    from microwakeword_b200.engine import MultiModelEngine
    torch = torch_cuda
    blobs = [_blob("hybrid"), _blob("int8"), _blob("generic_int8")]      # the three fresh-state fills; exact at any rotation
    SA = _S(torch)
    SB = SA + 91
    sets_a = [np.arange(0, SA, 2, dtype=np.int32), np.arange(1, SA, 3, dtype=np.int32), None]
    sets_b = [np.arange(0, SB, 3, dtype=np.int32), None, np.arange(2, SB, 2, dtype=np.int32)]
    A, R = MultiModelEngine(blobs, SA, streams=sets_a), MultiModelEngine(blobs, SA)
    B, twin = MultiModelEngine(blobs, SB, streams=sets_b), MultiModelEngine(blobs, SB, streams=sets_b)
    for e in (A, R):
        _serve(torch, e, 7, 10)
    for e in (B, twin):
        _serve(torch, e, 24, 50)                       # 17 live calls more: another rotation, the stride-17 model's pending rows again
    rng = np.random.default_rng(4)
    src, dst = rng.permutation(SA)[:200].astype(np.int32), rng.permutation(SB)[:200].astype(np.int32)
    rec = A.export_streams(src)
    masks = rec.data[:, :8].cpu().numpy().view(np.uint64).ravel()
    for k in range(3):
        member = np.isin(src, A.streams[k])
        assert np.array_equal((masks >> np.uint64(k)) & np.uint64(1), member.astype(np.uint64))
        if not member.all():                           # R: model k starts fresh on the sources that were not members
            R.set_streams(k, np.setdiff1d(np.arange(SA), src[~member]))
            R.set_streams(k, None)
    B.import_streams(dst, rec)

    def compare(i, n):
        a = _audio(torch, SA, n, 100 + i)
        b = _routed(torch, a, SB, 200 + i, src, dst)
        A.predict_clip(a)
        pr, pb, pt = R.predict_clip(a), B.predict_clip(b), twin.predict_clip(b)
        for k in range(3):
            rows_b = {int(s): j for j, s in enumerate(B.streams[k])}
            rows_t = {int(s): j for j, s in enumerate(twin.streams[k])}
            r, g, t = _bits(pr[k]), _bits(pb[k]), _bits(pt[k])
            moved = [(s, d) for s, d in zip(src, dst) if int(d) in rows_b and int(d) in members0[k]]
            assert len(moved) > 20
            assert np.array_equal(g[[rows_b[int(d)] for _, d in moved]], r[[s for s, _ in moved]]), (i, k)
            rest = [s for s in rows_t if s in rows_b and s not in moved_to]
            assert np.array_equal(g[[rows_b[s] for s in rest]], t[[rows_t[s] for s in rest]]), (i, k)

    members0 = [set(s.tolist()) for s in B.streams]    # the sets at import time
    moved_to = set(dst.tolist())
    for i, n in enumerate((480, 480, 4799, 480)):
        compare(i, n)
    # all streams for model 0 on both: the joiners start fresh, every earlier member keeps its compact row's state
    for e in (B, twin):
        e.set_streams(0, None)
    for i, n in enumerate((480, 4800, 480)):
        compare(10 + i, n)
    sb, st = B.state_dict(), twin.state_dict()
    rest = np.setdiff1d(np.arange(SB), dst)
    for key in ("carry", "estimate"):
        assert np.array_equal(sb[key][rest], st[key][rest])


# ---- the fp16 first-conv flag travels with the records -----------------------------------------------------------------------
def test_rows_flag_keeps_the_moved_stream_on_its_kernel(torch_cuda):
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    S = 300
    A, B = StreamEngine(_blob("f32"), S), StreamEngine(_blob("f32"), S + 5)
    g = torch.Generator(device="cuda").manual_seed(5)
    A.infer(3.0 * torch.randn(S, 3, 40, device="cuda", generator=g))           # rows of any value: the source's flag is clear
    rec = A.export_streams(np.arange(S))
    assert rec.layout.rows_are_features[0] == 0 and B.stream_layout().rows_are_features[0] == 1
    dst = np.arange(5, S + 5)
    B.import_streams(dst, rec)
    assert B.stream_layout().rows_are_features[0] == 0
    a = _audio(torch, S, 48000, 6)
    pa, pb = A.predict_clip(a), B.predict_clip(_routed(torch, a, S + 5, 7, np.arange(S), dst))
    assert pa.shape[1] == 99 and np.array_equal(_bits(pb)[dst], _bits(pa))


# ---- refusals: argument errors before any device work ---------------------------------------------------------------------------
def test_refusals_leave_the_destination_unchanged(torch_cuda):
    from microwakeword_b200.engine import MultiModelEngine, StreamEngine
    torch = torch_cuda
    S = 64
    f32, i8 = _blob("f32"), _blob("int8")

    def fresh(blob=f32):
        return StreamEngine(blob, S)

    def refused(dst, ids, rec, field, error=_lib.MwwError):
        before, count = dst.state_dict(), dst.launch_count
        with pytest.raises(error) as e:
            dst.import_streams(ids, rec)
        if error is _lib.MwwError:
            assert e.value.code == -1 and field in str(e.value), str(e.value)
        after = dst.state_dict()
        assert dst.launch_count == count
        for key in before:
            if key != "models":
                assert np.array_equal(before[key], after[key]), key

    ids = np.arange(8, dtype=np.int32)
    src = fresh()
    src.predict_clip(_audio(torch, S, 4801, 1))
    rec = src.export_streams(ids)
    match = fresh()
    match.predict_clip(_audio(torch, S, 4801, 2))
    refused(fresh(), ids, rec, "frontend_buffered")
    other = fresh(i8)
    other.predict_clip(_audio(torch, S, 4801, 2))
    refused(other, ids, rec, "model_hash of model 0")
    hop = fresh()
    hop.set_window_step(320)
    refused(hop, ids, fresh().export_streams(ids), "hop_samples")
    pend = fresh()
    pend.infer(torch.zeros(S, 1, 40, device="cuda"))
    refused(fresh(), ids, pend.export_streams(ids), "pending_rows of model 0")
    refused(MultiModelEngine([f32, f32], S), ids, fresh().export_streams(ids), "n_models")
    refused(match, np.asarray([1, 2, 1, 3, 4, 5, 6, 7], np.int32), rec, "listed twice")
    refused(match, np.asarray([1, 2, S, 3, 4, 5, 6, 7], np.int32), rec, "out of range")
    refused(match, np.asarray([1, 2, -1, 3, 4, 5, 6, 7], np.int32), rec, "out of range")
    from microwakeword_b200.engine import StreamRecords
    refused(match, ids[:7], rec, "", ValueError)                                            # one record too many
    refused(match, ids, StreamRecords(rec.data.cpu(), rec.layout), "", ValueError)           # host memory
    refused(match, ids, StreamRecords(rec.data.view(torch.int8), rec.layout), "", ValueError)
    refused(match, ids, StreamRecords(rec.data[:, :-16], rec.layout), "", ValueError)
    with pytest.raises(ValueError):
        match.export_streams(torch.arange(4, device="cuda"))
    with pytest.raises(_lib.MwwError):
        match.export_streams([0, S])
    # n == 0: nothing is launched, the layout is still filled and still checked
    count = match.launch_count
    empty = src.export_streams([])
    assert empty.data.shape == (0, rec.data.shape[1]) and bytes(empty.layout) == bytes(rec.layout)
    match.import_streams([], empty)
    assert match.launch_count == count
    refused(fresh(), np.zeros(0, np.int32), empty, "frontend_buffered")
    match.import_streams(ids, rec)                                                          # and the records that fit are taken
    assert np.array_equal(match.state_dict()["nn"][ids], src.state_dict()["nn"][ids])


# ---- save / load ----------------------------------------------------------------------------------------------------------------
def test_saved_records_import_like_the_originals(torch_cuda, tmp_path):
    from microwakeword_b200.engine import MultiModelEngine, StreamRecords
    torch = torch_cuda
    S = 200
    blobs = [_blob("f32"), _blob("generic_int8")]
    A, B, C = (MultiModelEngine(blobs, S) for _ in range(3))
    for e, seed in ((A, 1), (B, 2), (C, 2)):
        _serve(torch, e, 4, seed)
    src, dst = np.asarray([7, 150, 3, 99], np.int32), np.asarray([0, 199, 42, 7], np.int32)
    rec = A.export_streams(src)
    path = str(tmp_path / "streams.npz")
    rec.save(path)
    back = StreamRecords.load(path, "cuda:0")
    assert bytes(back.layout) == bytes(rec.layout) and torch.equal(back.data, rec.data)
    B.import_streams(dst, rec)
    C.import_streams(dst, back)
    a = _audio(torch, S, 4800, 9)
    for pb, pc in zip(B.predict_clip(a), C.predict_clip(a)):
        assert np.array_equal(_bits(pb), _bits(pc))


# ---- full size: growing a handle ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,SA,SB,shift", [("f32", 65536, 98304, 16384), ("int8", 65509, 65509 + 300, 150)])
def test_growing_a_handle_at_full_size(torch_cuda, kind, SA, SB, shift):
    """every stream of a full handle into a larger one: each copy kernel runs several waves past its grid (and, for 65 509
    streams, ends in a partial block)"""
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    A, B = StreamEngine(_blob(kind), SA), StreamEngine(_blob(kind), SB)
    for e, seed in ((A, 1), (B, 2)):
        for i in range(2):
            e.predict_clip(_audio(torch, e.n_streams, 48000, seed + 10 * i))
        for i in range(3):
            e.step(_audio(torch, e.n_streams, 480, seed + 30 + i))
    src = np.arange(SA, dtype=np.int32)
    dst = src + shift
    B.import_streams(dst, A.export_streams(src))
    for i, n in enumerate((48000, 480)):
        a = _audio(torch, SA, n, 60 + i)
        b = _audio(torch, SB, n, 70 + i)
        b[shift:shift + SA] = a
        pa, pb = A.predict_clip(a), B.predict_clip(b)
        assert torch.equal(pb[shift:shift + SA].view(torch.int32), pa.view(torch.int32)), (kind, n)
        del a, b, pa, pb


# ---- another GPU of the box -----------------------------------------------------------------------------------------------------
def test_records_pulled_to_a_peer_gpu(torch_cuda):
    import ctypes
    from microwakeword_b200.engine import StreamEngine, StreamRecords
    torch = torch_cuda
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU: moving records to a peer needs two")
    S = 500
    A, B = StreamEngine(_blob("f32"), S, device=0), StreamEngine(_blob("f32"), S, device=1)
    _serve(torch, A, 5, 1)
    with torch.cuda.device(1):
        for n in (4801,) + (480,) * 5:             # the source's rotation (fp32 live sums depend on it)
            B.predict_clip(_audio(torch, S, n, 2).to("cuda:1"))
    src, dst = np.arange(0, S, 2, dtype=np.int32), np.arange(1, S, 2, dtype=np.int32)
    rec = A.export_streams(src)
    a = _audio(torch, S, 480, 3)
    b = _routed(torch, a, S, 4, src, dst).to("cuda:1")
    torch.cuda.synchronize(0)
    pulled = torch.empty(rec.data.shape, dtype=torch.uint8, device="cuda:1")
    with torch.cuda.device(1):
        stream = ctypes.c_void_p(torch.cuda.current_stream(1).cuda_stream)
        _lib.check(None, _lib.lib().mww_copy_async(pulled.data_ptr(), rec.data.data_ptr(), pulled.numel(), stream))
        B.import_streams(dst, StreamRecords(pulled, rec.layout))
        pb = B.step(b)
    pa = A.step(a)
    assert np.array_equal(_bits(pb)[dst], _bits(pa)[src])
