"""G.711 audio on the GPU (run with -m gpu on an H100).

The contract of the _g711 entry points (include/mww.h): a call with mu-law or A-law bytes gives exactly what the int16 call
gives on the decoded samples -- bit-identical uint16 features, probabilities and state_dict() -- in every frontend kernel
that reads caller audio (fused clip at the benchmark's shape, K1 + K2, live fused, run-time hop, carry update), on the vector
and the scalar loads, from device, host (pinned and pageable) and remote-from-host memory, on multi-model handles with
stream sets, through the resampler at 8 kHz and with per-stream rates, and alternating with int16 and float32 calls on one
handle.  Every check below runs a G.711 handle beside an int16 twin fed the decoded samples.

Codes: P distinct base streams of uniformly random bytes (every code of the law), a third of them restricted to the quiet
segments; stream s carries base[s % P]."""

import ctypes
import os

import numpy as np
import pytest

import tflite_hybrid_writer as HW
from conftest import GOLDEN
from generic_range import GEOMETRIES, models as range_models
from microwakeword_b200 import _lib
from microwakeword_b200 import model_file as MF
from microwakeword_b200 import tflite_file as TF
from microwakeword_b200.engine import INPUT_RATES, MultiModelEngine, StreamEngine, inputs_for_rates
from test_g711 import alaw_ref, ulaw_ref

pytestmark = pytest.mark.gpu

P = 1021                       # prime: neighbouring CTAs' streams carry different audio
N_TOTAL = 100000
LAWS = ("ulaw", "alaw")
F32 = os.path.join(GOLDEN, "okay_nabu_synth_f32.mww")
I8 = os.path.join(GOLDEN, "okay_nabu_synth_int8.mww")


def _read(path):
    with open(path, "rb") as f:
        return f.read()


def model_blob(kind):
    if kind == "f32":
        return _read(F32)
    if kind == "int8":
        return _read(I8)
    if kind == "generic":
        return MF.write_container(range_models(GEOMETRIES["long_stride"])[0])
    assert kind == "hybrid"
    return MF.write_container(TF.tensors_from_tflite(HW.write_hybrid_mixednet(MF.load(F32), lambda op, n: n >= 1024, True)))


@pytest.fixture(scope="module")
def codes(torch_cuda):
    """{law: base codes uint8 [P, N_TOTAL] CUDA}, {law: their decoded samples int16 [P, N_TOTAL] CUDA}.  A call's rows are
    gathered from both with the same chunk(), so no test builds an index tensor as large as its audio.  At the end of the
    module the memory PyTorch cached for the 65 536-stream calls goes back to the device, where the library allocates its own
    buffers for the tests that follow."""
    import gc
    torch = torch_cuda
    rng = np.random.default_rng(711)
    raw = rng.integers(0, 256, (P, N_TOTAL), dtype=np.uint8)
    base, dec = {}, {}
    for law, quiet_bits, ref in (("ulaw", 0x70, ulaw_ref), ("alaw", 0x50, alaw_ref)):
        c = raw.copy()
        c[::3] = (c[::3] & 0x8F) | quiet_bits           # segment 0: the smallest steps of the law
        base[law] = torch.from_numpy(c).cuda()
        dec[law] = torch.from_numpy(ref(np.arange(256))[c]).cuda()
    yield base, dec
    del base, dec
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def chunk(torch, base, S, pos, n):
    idx = torch.arange(S, device="cuda") % P
    return base[:, pos:pos + n].index_select(0, idx).contiguous()


def with_layout(torch, x, offset, pitch):
    """x [S, n] -> the same values in a tensor whose storage starts `offset` elements in, with row pitch `pitch`"""
    S, n = x.shape
    flat = torch.full((S * pitch + offset,), 0x5A, dtype=x.dtype, device=x.device)
    view = flat[offset:offset + S * pitch].view(S, pitch)[:, :n]
    view.copy_(x)
    assert view.storage_offset() == offset and view.stride() == (pitch, 1)
    return view


def bits(torch, t):
    return t.contiguous().view({torch.float32: torch.int32, torch.uint16: torch.int16}[t.dtype])


def same_state(a, b, where="state"):
    if isinstance(a, dict):
        assert a.keys() == b.keys(), where
        for k in a:
            same_state(a[k], b[k], "%s.%s" % (where, k))
    elif isinstance(a, list):
        assert len(a) == len(b), where
        for i, (x, y) in enumerate(zip(a, b)):
            same_state(x, y, "%s[%d]" % (where, i))
    elif isinstance(a, np.ndarray):
        assert a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8)), where
    else:
        assert a == b, where


def same(torch, got, want, what):
    if isinstance(got, list):
        assert len(got) == len(want), what
        for k, (g, w) in enumerate(zip(got, want)):
            same(torch, g, w, "%s, model %d" % (what, k))
    elif isinstance(got, np.ndarray):
        assert got.shape == want.shape and np.array_equal(got.view(np.uint8), want.view(np.uint8)), what
    else:
        assert got.shape == want.shape and torch.equal(bits(torch, got), bits(torch, want)), what


def as_kind(torch, x_codes, dec, kind):
    """the call's audio on the G.711 side: the codes (a law), or the decoded samples as int16 or exact float32"""
    if kind in LAWS:
        return x_codes, kind
    if kind == "i16":
        return dec, None
    return dec.to(torch.float32) / 32768.0, None        # k / 2^15 is exact, and to_int16 of it is k again


def run_twins(torch, codes, S, blob, schedule, law="ulaw", hop=160, layout=None, rate=16000):
    """schedule: [(n_samples, kind)], kind a law or "i16" / "f32".  A model handle and a frontend-only handle take each call as
    `kind`; their twins take the decoded int16 samples.  Every call's probabilities and features and the final state of all
    four must be bit-identical."""
    base, decoded = codes
    engines = [StreamEngine(b, n_streams=S, input_rate=rate) for b in (blob, blob, None, None)]
    if hop != 160:
        for e in engines:
            e.set_window_step(hop)
    g, i, fg, fi = engines
    pos = 0
    for call, (n, kind) in enumerate(schedule):
        src = kind if kind in LAWS else law
        c, dec = chunk(torch, base[src], S, pos, n), chunk(torch, decoded[src], S, pos, n)
        x, call_law = as_kind(torch, c, dec, kind)
        if layout is not None:
            x = with_layout(torch, x, *layout(n))
        same(torch, g.predict_clip(x, law=call_law), i.predict_clip(dec), ("probabilities", call, n, kind))
        same(torch, fg.features(x, law=call_law), fi.features(dec), ("features", call, n, kind))
        pos += n
    assert pos <= N_TOTAL
    same_state(g.state_dict(), i.state_dict())
    same_state(fg.state_dict(), fi.state_dict())


CLIP = [(48000, "ulaw"), (16000, "alaw"), (4000, "ulaw")]                 # 3 s, 1 s entering with 320 buffered, 0.25 s
LIVE = [(480, law) for law in LAWS * 6]
BUFFERED = [(250, "ulaw"), (1000, "alaw"), (333, "alaw"), (16000, "ulaw"), (130, "ulaw"), (480, "alaw"), (480, "ulaw")]


@pytest.mark.parametrize("model", ["f32", "int8", "generic", "hybrid"])
def test_models_clip_live_and_buffered(torch_cuda, codes, model):
    run_twins(torch_cuda, codes, 2003, model_blob(model), CLIP + LIVE + BUFFERED)


def test_fused_clip_kernel_at_the_benchmark_shape(torch_cuda, codes):
    """3 s clips at 65 536 streams: the fused clip kernel, one CTA per stream"""
    run_twins(torch_cuda, codes, 65536, model_blob("f32"), [(48000, "ulaw"), (48000, "alaw")])


def test_k1_k2_kernels_below_the_fusing_stream_count(torch_cuda, codes):
    run_twins(torch_cuda, codes, 301, model_blob("int8"), CLIP + [(480, "alaw"), (480, "ulaw")])


def test_120_live_calls(torch_cuda, codes):
    run_twins(torch_cuda, codes, 4133, model_blob("f32"), [(480, LAWS[c % 7 % 2]) for c in range(120)])


def test_run_time_hop(torch_cuda, codes):
    run_twins(torch_cuda, codes, 1601, model_blob("f32"), [(16000, "ulaw"), (960, "alaw"), (480, "ulaw"), (3000, "alaw")], hop=320)


@pytest.mark.parametrize("where", ["vector", "byte_offset", "pitch_481", "buffered_not_8"])
def test_vector_and_scalar_loads(torch_cuda, codes, where):
    """8-byte-aligned bases with pitch, n_samples and buffered count multiples of 8 take the vector loads; a base one byte in,
    a pitch of 481 or a buffered count that is not a multiple of 8 take the scalar loads"""
    layout = {"vector": lambda n: (8, n + 8), "byte_offset": lambda n: (1, n), "pitch_481": lambda n: (0, max(481, n + 1)),
              "buffered_not_8": None}[where]
    sched = [(16000, "ulaw"), (480, "alaw"), (48000, "alaw"), (480, "ulaw"), (4000, "ulaw")]
    if where == "buffered_not_8":
        sched = [(100, "ulaw")] + sched                                    # 100 buffered, then 4 or 20 mod 8
    run_twins(torch_cuda, codes, 2003, model_blob("f32"), sched, layout=layout)


def test_all_four_sample_types_alternate_on_one_handle(torch_cuda, codes):
    kinds = ("i16", "ulaw", "f32", "alaw")
    sched = [(480, kinds[c % 4]) for c in range(12)] + [(16000, k) for k in kinds] + [(250, k) for k in kinds] + \
            [(480, kinds[(c + 1) % 4]) for c in range(8)]
    run_twins(torch_cuda, codes, 2003, model_blob("int8"), sched)


# ---- host and remote ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("law", LAWS)
def test_host_pinned_pageable_and_remote(torch_cuda, codes, law):
    torch = torch_cuda
    base, decoded = codes
    S = 4099
    blob = model_blob("f32")
    g, i = StreamEngine(blob, n_streams=S), StreamEngine(blob, n_streams=S)
    pos = 0
    for call, (n, path) in enumerate([(48000, "pageable"), (16000, "pinned"), (480, "pinned"), (4000, "remote0"), (480, "remote4"),
                                      (16000, "remote4"), (480, "pageable"), (480, "remote0")]):
        c = chunk(torch, base[law], S, pos, n)
        dec = chunk(torch, decoded[law], S, pos, n)
        c_np, dec_np = c.cpu().numpy(), dec.cpu().numpy()
        if path == "pageable":
            same(torch, g.predict_clip_host(c_np, law=law), i.predict_clip_host(dec_np), (path, call))
        elif path == "pinned":
            hc, hd = g.host_buffer(c_np.shape, np.uint8), i.host_buffer(dec_np.shape, np.int16)
            hc[:], hd[:] = c_np, dec_np
            same(torch, g.predict_clip_host(hc, law=law), i.predict_clip_host(hd), (path, call))
        else:
            tiles = int(path[-1])
            hc, hd = g.host_buffer(c_np.shape, np.uint8), i.host_buffer(dec_np.shape, np.int16)
            hc[:], hd[:] = c_np, dec_np
            got = g.predict_clip_remote(hc.ctypes.data, n, tiles=tiles, dtype=np.uint8, law=law)
            want = i.predict_clip_remote(hd.ctypes.data, n, tiles=tiles, dtype=np.int16)
            torch.cuda.synchronize()
            same(torch, got, want, (path, call))
        pos += n
    same_state(g.state_dict(), i.state_dict())


def test_multi_model_with_stream_sets_device_and_host(torch_cuda, codes):
    torch = torch_cuda
    base, decoded = codes
    S = 3001
    rng = np.random.default_rng(3)
    subset = np.flatnonzero(rng.random(S) < 0.4).astype(np.int32)
    blobs = [model_blob("f32"), model_blob("int8"), model_blob("generic")]
    streams = [None, subset, subset[::3]]
    g, i = MultiModelEngine(blobs, S, streams=streams), MultiModelEngine(blobs, S, streams=streams)
    pos = 0
    for call, (n, law, path) in enumerate([(16000, "ulaw", "device"), (480, "alaw", "device"), (48000, "alaw", "host"),
                                           (480, "ulaw", "host"), (480, "ulaw", "device"), (4000, "alaw", "remote")]):
        c = chunk(torch, base[law], S, pos, n)
        dec = chunk(torch, decoded[law], S, pos, n)
        if path == "device":
            same(torch, g.predict_clip(c, law=law), i.predict_clip(dec), (path, call))
        elif path == "host":
            same(torch, g.predict_clip_host(c.cpu().numpy(), law=law), i.predict_clip_host(dec.cpu().numpy()), (path, call))
        else:
            hc, hd = g.host_buffer(tuple(c.shape), np.uint8), i.host_buffer(tuple(dec.shape), np.int16)
            hc[:], hd[:] = c.cpu().numpy(), dec.cpu().numpy()
            got = g.predict_clip_remote(hc.ctypes.data, n, tiles=4, dtype=np.uint8, law=law)
            want = i.predict_clip_remote(hd.ctypes.data, n, tiles=4)
            torch.cuda.synchronize()
            same(torch, got, want, (path, call))
        pos += n
    same_state(g.state_dict(), i.state_dict())


# ---- resampling ------------------------------------------------------------------------------------------------------------
def test_8khz_clips_and_live_calls(torch_cuda, codes):
    run_twins(torch_cuda, codes, 2003, model_blob("f32"),
              [(24000, "ulaw"), (8000, "alaw"), (1001, "ulaw")] + [(240, LAWS[c % 2]) for c in range(20)], rate=8000)


@pytest.mark.parametrize("law", LAWS)
def test_per_stream_rates_all_seven(torch_cuda, codes, law):
    torch = torch_cuda
    base, decoded = codes
    rng = np.random.default_rng(17)
    S = 2003
    rates = np.asarray(INPUT_RATES, np.int32)[rng.integers(0, len(INPUT_RATES), S)]
    rates[:len(INPUT_RATES)] = INPUT_RATES
    blob = model_blob("int8")
    g, i = StreamEngine(blob, n_streams=S, stream_rates=rates), StreamEngine(blob, n_streams=S, stream_rates=rates)
    fg, fi = StreamEngine(None, n_streams=S, stream_rates=rates), StreamEngine(None, n_streams=S, stream_rates=rates)
    splits = [480] * 4 + [int(2 * rng.integers(1, 2000)) for _ in range(6)] + [480] * 4
    t = 0
    pos = 0
    for call, n16 in enumerate(splits):
        D = inputs_for_rates(rates, t, n16)
        width = int(D.max())
        c = chunk(torch, base[law], S, pos, width + 3)[:, :width]          # padding past D_s: bytes the library must not read
        dec = chunk(torch, decoded[law], S, pos, width + 3)[:, :width]
        same(torch, g.predict_clip(c, samples16=n16, law=law), i.predict_clip(dec, samples16=n16), ("probabilities", call, n16))
        same(torch, fg.features(c, samples16=n16, law=law), fi.features(dec, samples16=n16), ("features", call, n16))
        t += n16
        pos += width
    assert pos <= N_TOTAL
    for a, b in ((g, i), (fg, fi)):
        same_state(a.state_dict(), b.state_dict())


# ---- refusals ----------------------------------------------------------------------------------------------------------------
def test_unknown_laws_leave_the_handle_unchanged(torch_cuda, codes):
    torch = torch_cuda
    base, _ = codes
    S = 64
    e = StreamEngine(model_blob("f32"), n_streams=S)
    e.predict_clip(chunk(torch, base["ulaw"], S, 0, 1000), law="ulaw")
    before = e.state_dict()
    L, h = e._L, e._h
    c = chunk(torch, base["alaw"], S, 0, 480)
    host = c.cpu().numpy()
    feat = torch.empty((S, 8, 40), dtype=torch.uint16, device="cuda")
    probs = torch.empty((S, 8), dtype=torch.float32, device="cuda")
    probs_h = np.empty((S, 8), np.float32)
    got = ctypes.c_int(0)
    ptrs = (ctypes.c_void_p * 1)(probs.data_ptr())
    ptrs_h = (ctypes.c_void_p * 1)(probs_h.ctypes.data)
    maxp = (ctypes.c_int * 1)(8)
    st = e._cu_stream()
    for law in (0, 3, -1):
        calls = [
            L.mww_features_g711(h, c.data_ptr(), law, 480, 480, feat.data_ptr(), 8, ctypes.byref(got), st),
            L.mww_predict_clip_g711(h, c.data_ptr(), law, 480, 480, probs.data_ptr(), 8, ctypes.byref(got), st),
            L.mww_predict_clip_host_g711(h, host.ctypes.data, law, 480, 480, probs_h.ctypes.data, 8, ctypes.byref(got)),
            L.mww_predict_clip_remote_g711(h, host.ctypes.data, law, 480, 480, probs.data_ptr(), 8, ctypes.byref(got), 4, st),
            L.mww_predict_clip_multi_g711(h, c.data_ptr(), law, 480, 480, ptrs, maxp, None, st),
            L.mww_predict_clip_host_multi_g711(h, host.ctypes.data, law, 480, 480, ptrs_h, maxp, None),
            L.mww_predict_clip_remote_multi_g711(h, host.ctypes.data, law, 480, 480, ptrs, maxp, None, 0, st),
        ]
        assert calls == [-1] * 7, (law, calls)          # MWW_EINVAL
        assert b"law" in L.mww_last_error(h)
    torch.cuda.synchronize()
    same_state(e.state_dict(), before)
    # the handle still works, and continues exactly like a twin that never saw the refusals
    twin = StreamEngine(model_blob("f32"), n_streams=S)
    twin.predict_clip(chunk(torch, base["ulaw"], S, 0, 1000), law="ulaw")
    same(torch, e.predict_clip(c, law="alaw"), twin.predict_clip(c, law="alaw"), "after refusals")


def test_one_model_entry_points_refuse_several_models(torch_cuda, codes):
    torch = torch_cuda
    base, _ = codes
    S = 64
    e = MultiModelEngine([model_blob("f32"), model_blob("int8")], S)
    before = e.state_dict()
    L, h = e._L, e._h
    c = chunk(torch, base["ulaw"], S, 0, 480)
    host = c.cpu().numpy()
    probs = torch.empty((S, 8), dtype=torch.float32, device="cuda")
    probs_h = np.empty((S, 8), np.float32)
    got = ctypes.c_int(0)
    st = e._cu_stream()
    for law in (_lib.MWW_G711_ULAW, _lib.MWW_G711_ALAW):
        rcs = [L.mww_predict_clip_g711(h, c.data_ptr(), law, 480, 480, probs.data_ptr(), 8, ctypes.byref(got), st),
               L.mww_predict_clip_host_g711(h, host.ctypes.data, law, 480, 480, probs_h.ctypes.data, 8, ctypes.byref(got)),
               L.mww_predict_clip_remote_g711(h, host.ctypes.data, law, 480, 480, probs.data_ptr(), 8, ctypes.byref(got), 0, st)]
        assert rcs == [-1] * 3
        assert b"_multi_g711" in L.mww_last_error(h)
    torch.cuda.synchronize()
    same_state(e.state_dict(), before)
