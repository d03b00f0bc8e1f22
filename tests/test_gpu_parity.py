"""GPU parity tests (run with -m gpu on an H100).  Every call goes through the C-ABI of
include/mww.h (via microwakeword_b200.engine / .inference) and is compared with the CPU oracle on the
same seeded inputs and with the committed golden fixtures.

Bars: uint16 features bit-exact; int8 model bit-exact; fp32 probabilities within 1e-5 of the fp32
oracle (north_star allows 1e-3; the only difference is fma / summation order)."""

import os

import numpy as np
import pytest

import oracle
from conftest import GOLDEN, edge_case_audio, synth_audio

pytestmark = pytest.mark.gpu

F32_TOL = 1e-5


def _blob(name):
    with open(os.path.join(GOLDEN, name), "rb") as f:
        return f.read()


def _u16(t):
    import torch
    return t.view(torch.int16).cpu().numpy().view(np.uint16)


def _dev_u16(a, torch):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int16)).cuda().view(torch.uint16)


def test_library_loaded_and_device_is_hopper(torch_cuda):
    from microwakeword_b200 import _lib
    assert os.path.exists(_lib.SO_PATH)
    L = _lib.lib()
    for sym in _lib.EXPORTS:
        assert hasattr(L, sym)
    assert torch_cuda.cuda.get_device_capability(0) == (9, 0)      # the library is built for sm_90a only


def test_features_bit_exact_random_and_edge(torch_cuda):
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    audio = np.concatenate([np.stack([synth_audio(16000, 200 + i) for i in range(50)]), edge_case_audio(16000)])
    eng = StreamEngine(None, n_streams=audio.shape[0])
    got = _u16(eng.features(torch.from_numpy(audio).cuda()))
    want, _ = oracle.run_pipeline(None, audio, want_probs=False, threads=8)
    assert got.shape == want.shape == (audio.shape[0], 98, 40)
    assert np.array_equal(got, want)
    assert eng.frontend_buffered == 320


def test_features_golden_config0(torch_cuda):
    from microwakeword_b200.audio.audio_utils import generate_features_for_clip
    clip = np.load(os.path.join(GOLDEN, "config0_audio.npy"))
    want = np.load(os.path.join(GOLDEN, "config0_features.npy"))
    got = generate_features_for_clip(clip)                      # float32 = uint16 * 0.0390625
    assert got.dtype == np.float32 and got.shape == (997, 40)
    assert np.array_equal(got, want.astype(np.float32) * np.float32(0.0390625))
    got_tf = generate_features_for_clip(clip, step_ms=10, use_c=False)   # TF-op semantics: all 998 windows, uint16
    assert got_tf.dtype == np.uint16 and got_tf.shape == (998, 40)
    assert np.array_equal(got_tf[:997], want)
    # float input path (audio_utils.py:47-48)
    got_f = generate_features_for_clip(clip.astype(np.float32) / 32768.0)
    assert np.array_equal(got_f, got)


def test_features_chunking_invariance_and_state(torch_cuda):
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    audio = np.stack([synth_audio(24000, 300 + i) for i in range(9)])
    whole, _ = oracle.run_pipeline(None, audio, want_probs=False)
    eng = StreamEngine(None, n_streams=9)
    rng = np.random.default_rng(4)
    pos, parts = 0, []
    while pos < audio.shape[1]:
        n = int(rng.integers(1, 1500))
        chunk = np.ascontiguousarray(audio[:, pos:pos + n])
        parts.append(_u16(eng.features(torch.from_numpy(chunk).cuda())))
        pos += chunk.shape[1]
    got = np.concatenate(parts, 1)
    assert np.array_equal(got, whole)
    # state equals the oracle's after the same audio
    st = eng.state_dict()
    fe = oracle.Frontend()
    fe.stream(audio[3])
    buf, used, est = fe.state()
    assert st["frontend_buffered"] == used
    assert np.array_equal(st["carry"][3][:used], buf[:used])
    assert np.array_equal(st["estimate"][3], est)


def test_fused_short_call_frontend(torch_cuda):
    """Hop-aligned short calls (1..8 frames, exactly 2 hops left over) take the fused K1+K2+carry kernel: every frames-per-call
    count, stream counts that do not fill the last CTA, aligned and unaligned audio views, against the oracle and against the
    same engine with the fusion switched off."""
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    S = 37
    calls = [480] + [160 * k for k in (1, 2, 3, 4, 5, 6, 7, 8, 3, 3, 1, 8)] + [2000, 160, 480]      # 2000: not hop aligned -> unfused, then re-aligns? no: stays off the grid
    total = sum(calls) + 160 * 4
    audio = np.concatenate([np.stack([synth_audio(total, 1500 + i) for i in range(S - 3)]), edge_case_audio(total)[:3]])
    whole, _ = oracle.run_pipeline(None, audio, want_probs=False)
    dev = torch.from_numpy(audio).cuda()
    pad = torch.zeros((S, total + 3), dtype=torch.int16, device="cuda")
    pad[:, 3:] = dev                                                       # rows start 6 bytes off 16-byte alignment -> scalar staging path
    os.environ["MWW_NO_FUSE"] = "1"
    try:
        plain = StreamEngine(None, n_streams=S)
    finally:
        del os.environ["MWW_NO_FUSE"]
    for name, src, off in (("aligned", dev, 0), ("unaligned", pad, 3)):
        eng = StreamEngine(None, n_streams=S)
        plain.reset()
        pos, parts, launches = 0, [], []
        for n in calls:
            l0 = eng.launch_count
            view = src[:, off + pos:off + pos + n]
            a = eng.features(view if name == "unaligned" else view.contiguous())
            b = plain.features(dev[:, pos:pos + n].contiguous())
            assert bool((a.view(torch.int16) == b.view(torch.int16)).all()), (name, n)
            parts.append(_u16(a))
            launches.append(eng.launch_count - l0)
            pos += n
        got = np.concatenate(parts, 1)
        assert np.array_equal(got, whole[:, :got.shape[1]]), name
        assert launches[:13] == [1] * 13 and launches[13] == 3, launches           # one fused launch per aligned call; K1 + K2 + carry otherwise
        sa, sb = eng.state_dict(), plain.state_dict()
        assert np.array_equal(sa["carry"], sb["carry"]) and np.array_equal(sa["estimate"], sb["estimate"])


@pytest.mark.parametrize("kind", ["f32", "int8"])
def test_model_golden_config0(torch_cuda, kind):
    from microwakeword.inference import Model               # the reference's import path
    m = Model(os.path.join(GOLDEN, "okay_nabu_synth_%s.mww" % kind))
    assert m.is_quantized_model == (kind == "int8") and m.input_feature_slices == 3 and m.stride == 3
    feats = np.load(os.path.join(GOLDEN, "config0_features.npy"))
    want = np.load(os.path.join(GOLDEN, "config0_probs_%s.npy" % kind))
    got = m.predict_spectrogram(feats)
    assert isinstance(got, list) and len(got) == 332 and isinstance(got[0], np.float32)
    if kind == "int8":
        assert np.array_equal(np.asarray(got), want)
    else:
        assert np.abs(np.asarray(got) - want).max() <= F32_TOL
    # state persists across calls (inference.py never resets; SURVEY.md 3.3 item 5): a second pass differs from a fresh one
    again = np.asarray(m.predict_spectrogram(feats[:30]))
    m.reset()
    fresh = np.asarray(m.predict_spectrogram(feats[:30]))
    assert np.array_equal(fresh, np.asarray(got[:10])) if kind == "int8" else np.abs(fresh - np.asarray(got[:10])).max() <= F32_TOL
    assert not np.array_equal(again, fresh)
    # predict_clip = fresh frontend + NN (state carried): after reset equals the golden chain
    m.reset()
    clip = np.load(os.path.join(GOLDEN, "config0_audio.npy"))
    pc = np.asarray(m.predict_clip(clip))
    assert pc.shape == (332,)
    assert np.array_equal(pc, want) if kind == "int8" else np.abs(pc - want).max() <= F32_TOL


def test_predict_spectrogram_dtypes_and_quirks(torch_cuda):
    from microwakeword_b200.inference import Model
    feats = np.load(os.path.join(GOLDEN, "config0_features.npy"))[:92]
    m = Model(os.path.join(GOLDEN, "okay_nabu_synth_f32.mww"))
    a = np.asarray(m.predict_spectrogram(feats)); m.reset()
    b = np.asarray(m.predict_spectrogram(feats.astype(np.float32) * np.float32(0.0390625))); m.reset()
    c = np.asarray(m.predict_spectrogram(feats.astype(np.float64) * 0.0390625)); m.reset()
    # 92 rows -> 30 chunks, 2 rows dropped.  uint16 rows take the wgmma clip kernel, float rows the mma.sync one: same values up
    # to the order of fp32 additions inside the two tensor-core paths; float32 and float64 rows are the same path, bit for bit
    assert len(a) == 30 and np.abs(a - b).max() <= 2e-6 and np.array_equal(b, c)
    assert m.predict_spectrogram(feats[:2]) == []
    # stride 1: overlapping chunks, each is one invoke (inference.py:98-105)
    m1 = Model(os.path.join(GOLDEN, "okay_nabu_synth_f32.mww"), stride=1)
    got = np.asarray(m1.predict_spectrogram(feats[:12]))
    from oracle import mixednet_ref as R
    from microwakeword_b200 import model_file as MF
    om = R.FoldedStreamingF32(MF.load(os.path.join(GOLDEN, "okay_nabu_synth_f32.mww")))
    want = np.asarray(R.predict_spectrogram(om, feats[:12], stride=1))
    assert got.shape == want.shape == (10,) and np.abs(got - want).max() <= F32_TOL
    # int8 model: float rows are quantised with the truncating rule; pre-quantised int8 rows bypass it (inference.py:110)
    q = Model(os.path.join(GOLDEN, "okay_nabu_synth_int8.mww"))
    pa = np.asarray(q.predict_spectrogram(feats)); q.reset()
    rows_q = q.quantize_input_data(feats.astype(np.float32) * np.float32(0.0390625), q.input_details[0])
    assert rows_q.dtype == np.int8
    pb = np.asarray(q.predict_spectrogram(rows_q))
    assert np.array_equal(pa, pb)
    assert q.dequantize_output_data(np.uint8(255), q.output_details[0]) == np.float32(1.0)


@pytest.mark.parametrize("kind", ["f32", "int8"])
def test_batch_pipeline_device_and_host_paths(torch_cuda, kind):
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    blob = _blob("okay_nabu_synth_%s.mww" % kind)
    audio = np.concatenate([np.stack([synth_audio(30000, 400 + i) for i in range(40)]), edge_case_audio(30000)])
    _, want = oracle.run_pipeline(blob, audio, want_features=False, threads=8)
    S = audio.shape[0]
    eng = StreamEngine(blob, n_streams=S)
    got = eng.predict_clip(torch.from_numpy(audio).cuda()).cpu().numpy()
    assert got.shape == want.shape
    ok = np.array_equal(got, want) if kind == "int8" else np.abs(got - want).max() <= F32_TOL
    assert ok
    # host-buffer path with forced small tiles -> many pipelined tiles, same answer
    os.environ["MWW_SCRATCH_MB"] = "1"
    try:
        eng2 = StreamEngine(blob, n_streams=S)
    finally:
        del os.environ["MWW_SCRATCH_MB"]
    got2 = eng2.predict_clip_host(audio)
    assert np.array_equal(got2, got)
    # live-step mode: 480 new samples per call == the clip result
    eng3 = StreamEngine(blob, n_streams=S)
    dev = torch.from_numpy(audio).cuda()
    parts = [eng3.step(dev[:, i:i + 480].contiguous()) for i in range(0, audio.shape[1] - 479, 480)]
    got3 = torch.cat(parts, 1).cpu().numpy()
    n = got3.shape[1]
    assert n >= want.shape[1] - 1
    # int8: one integer kernel either way -> identical; fp32: the 3-row calls take the stream-parallel live-step kernel,
    # whose summation order differs from the clip kernel's
    assert np.array_equal(got3, got[:, :n]) if kind == "int8" else np.abs(got3 - want[:, :n]).max() <= F32_TOL


def test_golden_batch_fixture(torch_cuda):
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    audio = np.load(os.path.join(GOLDEN, "batch_audio.npy"))
    eng = StreamEngine(_blob("okay_nabu_synth_int8.mww"), n_streams=audio.shape[0])
    assert np.array_equal(eng.predict_clip(torch.from_numpy(audio).cuda()).cpu().numpy(), np.load(os.path.join(GOLDEN, "batch_probs_int8.npy")))
    eng = StreamEngine(_blob("okay_nabu_synth_f32.mww"), n_streams=audio.shape[0])
    got = eng.predict_clip(torch.from_numpy(audio).cuda()).cpu().numpy()
    assert np.abs(got - np.load(os.path.join(GOLDEN, "batch_probs_f32.npy"))).max() <= F32_TOL
    fe = StreamEngine(None, n_streams=audio.shape[0])
    assert np.array_equal(_u16(fe.features(torch.from_numpy(audio).cuda())), np.load(os.path.join(GOLDEN, "batch_features.npy")))


def test_nn_state_roundtrip_and_reset_ids(torch_cuda):
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    blob = _blob("okay_nabu_synth_f32.mww")
    audio = np.stack([synth_audio(20000, 500 + i) for i in range(5)])
    dev = torch.from_numpy(audio).cuda()
    a = StreamEngine(blob, n_streams=5)
    first = a.predict_clip(dev[:, :9000].contiguous()).cpu().numpy()
    snap = a.state_dict()
    rest = a.predict_clip(dev[:, 9000:].contiguous()).cpu().numpy()
    b = StreamEngine(blob, n_streams=5)
    b.load_state_dict(snap)
    assert np.array_equal(b.predict_clip(dev[:, 9000:].contiguous()).cpu().numpy(), rest)
    _, whole = oracle.run_pipeline(blob, audio, want_features=False)
    assert np.abs(np.concatenate([first, rest], 1) - whole).max() <= F32_TOL
    # per-stream reset zeroes that stream's state only
    a.reset([2])
    st = a.state_dict()
    assert not st["nn"][2].any() and not st["estimate"][2].any() and st["nn"][1].any()


@pytest.mark.parametrize("kind", ["f32", "int8", "f32_v1", "f32_v2"])
def test_live_rings_rotate_and_canonicalise(torch_cuda, kind, monkeypatch):
    if kind.startswith("f32_v"):   # the default is variant 3 (bulk-copy stages); 1 and 2 stay as references (MWW_LIVE_VARIANT is read at mww_create)
        monkeypatch.setenv("MWW_LIVE_VARIANT", kind[-1])
        kind = "f32"
    """Live calls keep the NN rings rotated (only the new row is written); a snapshot, a clip call or a mode switch
    rotates them back.  Every hand-over must continue the same probability chain as the oracle."""
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    blob = _blob("okay_nabu_synth_%s.mww" % kind)
    exact = kind == "int8"                                       # integer path: bit-exact through every hand-over
    S = 70                                                       # 2 full groups of 32 streams + a ragged one
    audio = np.stack([synth_audio(48000, 1200 + i) for i in range(S)])
    _, whole = oracle.run_pipeline(blob, audio, want_features=False, threads=8)
    dev = torch.from_numpy(audio).cuda()
    live = StreamEngine(blob, n_streams=S)
    clip = StreamEngine(blob, n_streams=S)
    got, pos = [], 0
    for n_live in (23, 1, 40):                                   # 23, 24 and 64 live steps: every ring wraps at least once (rows 4..22)
        for _ in range(n_live):
            got.append(live.step(dev[:, pos:pos + 480].contiguous()))
            pos += 480
        # (a) snapshot == state of an engine that only ever ran the clip kernel over the same samples
        clip.reset()
        clip.predict_clip(dev[:, :pos].contiguous())
        a, b = live.state_dict(), clip.state_dict()
        assert np.array_equal(a["nn"], b["nn"]) if exact else np.abs(a["nn"] - b["nn"]).max() <= 1e-4
        assert np.array_equal(a["pending"], b["pending"]) and np.array_equal(a["carry"], b["carry"])
        # (b) a longer call goes through the clip kernel, then live again
        got.append(live.predict_clip(dev[:, pos:pos + 2000].contiguous()))
        pos += 2000
    # (c) per-stream reset while the rings are rotated, then keep stepping: stream 3 restarts from silence
    for _ in range(5):
        got.append(live.step(dev[:, pos:pos + 480].contiguous()))
        pos += 480
    got = torch.cat(got, 1).cpu().numpy()
    assert np.array_equal(got, whole[:, :got.shape[1]]) if exact else np.abs(got - whole[:, :got.shape[1]]).max() <= F32_TOL
    live.reset([3])
    st = live.state_dict()
    fresh = StreamEngine(blob, n_streams=1).state_dict()["nn"][0]          # fp32: zeros; int8: the zero points
    assert np.array_equal(st["nn"][3], fresh) and not np.array_equal(st["nn"][4], fresh)
    # (d) loading a snapshot into a rotated engine resets the rotation
    live.step(dev[:, :480].contiguous())
    live.load_state_dict(clip.state_dict())
    x = live.step(dev[:, pos:pos + 480].contiguous())
    clip2 = StreamEngine(blob, n_streams=S)
    clip2.load_state_dict(clip.state_dict())
    assert np.abs((x - clip2.step(dev[:, pos:pos + 480].contiguous())).cpu().numpy()).max() <= (0 if exact else 1e-5)


def test_errors_are_loud(torch_cuda):
    from microwakeword_b200 import _lib
    from microwakeword_b200.engine import StreamEngine
    with pytest.raises(_lib.MwwError):
        StreamEngine(b"not a model", n_streams=1)
    eng = StreamEngine(None, n_streams=2)
    with pytest.raises(_lib.MwwError):
        eng.infer(torch_cuda.zeros((2, 3, 40), dtype=torch_cuda.float32, device="cuda"))
    with pytest.raises(ValueError):
        eng.features(torch_cuda.zeros((3, 480), dtype=torch_cuda.int16, device="cuda"))


def test_full_size_properties(torch_cuda):
    """BASELINE.json configs[1] scale (65 536 streams), checked through size-independent properties:
    replicated streams give identical outputs, silence gives the model's fixed silence response,
    a sample of streams matches the oracle, and chunked == whole."""
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    S, N = 65536, 4800
    base = np.concatenate([np.stack([synth_audio(N, 600 + i) for i in range(60)]), edge_case_audio(N)[:4]])   # 64 distinct streams
    reps = S // base.shape[0]
    dev = torch.from_numpy(base).cuda().repeat(reps, 1)
    blob = _blob("okay_nabu_synth_int8.mww")
    eng = StreamEngine(blob, n_streams=S)
    got = eng.predict_clip(dev)
    assert got.shape == (S, 9)
    g = got.view(reps, base.shape[0], 9)
    assert bool((g == g[0:1]).all())                      # every replica identical -> no cross-stream leakage
    _, want = oracle.run_pipeline(blob, base, want_features=False, threads=8)
    assert np.array_equal(g[0].cpu().numpy(), want)
    # chunked streaming at full size equals the whole-clip call
    eng.reset()
    a = eng.predict_clip(dev[:, :1760].contiguous())
    b = eng.predict_clip(dev[:, 1760:].contiguous())
    assert bool((torch.cat([a, b], 1) == got).all())


def test_feature_extractor_only_config3(torch_cuda):
    """BASELINE.json configs[3]: 1 M 30 ms windows through the frontend alone, both layouts SURVEY.md 8(d) names --
    4 096 streams x 256 frames with carried state, and 1 048 576 stateless windows of 480 samples (the packed short-call
    kernel).  Distinct content is replicated so that full size is checked through replica equality + an oracle sample."""
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    # streaming layout
    S, F = 4096, 256
    N = 160 * F + 320
    base = np.stack([synth_audio(N, 900 + i) for i in range(32)])
    dev = torch.from_numpy(base).cuda().repeat(S // 32, 1)
    eng = StreamEngine(None, n_streams=S)
    got = eng.features(dev)
    assert got.shape == (S, F, 40)
    g = got.view(torch.int16).view(S // 32, 32, F, 40)
    assert bool((g == g[0:1]).all())
    for i in (0, 7, 31):
        assert np.array_equal(g[0, i].cpu().numpy().view(np.uint16), oracle.Frontend().stream(base[i]))
    del eng, dev, got, g
    # stateless layout: every 480-sample window from the reset state -> exactly one row each
    W = 1 << 20
    wins = np.stack([synth_audio(480, 2000 + i) for i in range(1020)] + list(edge_case_audio(480)[:4]))    # 1024 distinct windows
    devw = torch.from_numpy(wins).cuda().repeat(W // 1024, 1)
    engw = StreamEngine(None, n_streams=W)
    out = torch.empty((W, 1, 40), dtype=torch.uint16, device="cuda")
    gw = engw.features(devw, out=out)
    assert gw.shape == (W, 1, 40) and gw.data_ptr() == out.data_ptr()
    gv = gw.view(torch.int16).view(W // 1024, 1024, 40)
    assert bool((gv == gv[0:1]).all())
    want = np.stack([oracle.Frontend().stream(w)[0] for w in wins])
    assert np.array_equal(gv[0].cpu().numpy().view(np.uint16), want)


def test_ragged_batch_feature_generation(torch_cuda):
    """SURVEY.md 8 f-3 caller: many clips of different lengths through one frontend launch == one clip at a time."""
    from microwakeword_b200.audio.audio_utils import generate_features_for_clips
    lengths = [16000, 480, 479, 641, 24000, 8000, 16001, 0, 12345]
    clips = [synth_audio(max(n, 1), 700 + i)[:n] for i, n in enumerate(lengths)]
    got = generate_features_for_clips(clips)
    assert len(got) == len(clips)
    for c, g in zip(clips, got):
        want = oracle.generate_features_for_clip(c)
        assert g.dtype == np.float32 and g.shape == want.shape
        assert np.array_equal(g, want.astype(np.float32) * np.float32(0.0390625))
    got_tf = generate_features_for_clips(clips, use_c=False)
    for c, g in zip(clips, got_tf):
        fe = oracle.Frontend()
        assert g.dtype == np.uint16 and np.array_equal(g, fe.stream(c))


def test_nonstreaming_batch_equals_keras_nonstreaming_graph(torch_cuda):
    """SURVEY.md 8 f-4: batched non-streaming evaluation through the clip kernel == the whole-clip 'valid' graph."""
    from microwakeword_b200 import model_file as MF
    from microwakeword_b200.inference import Model
    from oracle import mixednet_ref as R
    path = os.path.join(GOLDEN, "okay_nabu_synth_f32.mww")
    m = Model(path)
    feats = np.load(os.path.join(GOLDEN, "config0_features.npy"))
    windows = np.stack([feats[s:s + 204] for s in (0, 37, 200, 555, 793)])          # [5, 204, 40] uint16
    got = m.predict_nonstreaming(windows)
    t = MF.load(path)
    want = np.asarray([R._sigmoid(R.nonstreaming_logits(t, w.astype(np.float32) * R.FEATURE_SCALE)[-1]) for w in windows])
    assert got.shape == (5,) and np.abs(got - want).max() <= F32_TOL
    with pytest.raises(ValueError):
        m.predict_nonstreaming(windows[:, :100])


def _single_rank_group(torch):
    import socket

    import torch.distributed as dist
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    dist.init_process_group("nccl", init_method="tcp://127.0.0.1:%d" % port, rank=0, world_size=1, device_id=torch.device("cuda", 0))
    return dist


@pytest.mark.parametrize("kind", ["f32", "int8"])
def test_staged_remote_path_equals_resident_path_and_oracle(torch_cuda, kind, monkeypatch):
    """mww_predict_clip_remote with a source this GPU has to DMA from (pinned host memory stands in for a peer GPU's buffer
    on a one-GPU box): ragged tiles 4,4,4,1, two staging buffers, scores written straight into the device output --
    identical to the resident path, across two consecutive calls (state carried), and to the oracle."""
    from microwakeword_b200.engine import StreamEngine, host_array
    torch = torch_cuda
    monkeypatch.setenv("MWW_MIN_TILE_STREAMS", "1")
    blob = _blob("okay_nabu_synth_%s.mww" % kind)
    audio = np.stack([synth_audio(9600, 900 + i) for i in range(13)])
    pinned = host_array(audio.shape, np.int16, 0)
    pinned[:] = audio
    dev = torch.from_numpy(audio).cuda()
    one = StreamEngine(blob, n_streams=13)
    staged = StreamEngine(blob, n_streams=13)
    for call in range(2):
        want = one.predict_clip(dev)
        got = staged.predict_clip_remote(pinned.ctypes.data, 9600, tiles=4)
        assert got.shape == want.shape and torch.equal(got, want), call
    _, ref = oracle.run_pipeline(blob, np.concatenate([audio, audio], 1), want_features=False)
    err = np.abs(want.cpu().numpy() - ref[:, -want.shape[1]:]).max()           # the second call's steps are the last ones
    assert (err == 0.0) if kind == "int8" else (err <= F32_TOL)
    # the tile timeline of a profiled staged call: 4 tiles, each copy before its kernels, copies and kernels in tile order;
    # profiling must not change the result
    staged.profile(True)
    third = one.predict_clip(dev)
    again = staged.predict_clip_remote(pinned.ctypes.data, 9600, tiles=4)
    tl = staged.timeline_read()
    staged.profile_read()
    staged.profile(False)
    assert torch.equal(again, third)
    assert tl.shape == (4, 4) and tl[0, 0] == 0.0 and (tl >= 0).all()
    assert (tl[:, 0] <= tl[:, 1]).all() and (tl[:, 1] <= tl[:, 3]).all() and (tl[:, 2] <= tl[:, 3]).all()
    assert (np.diff(tl[:, 1]) >= 0).all() and (np.diff(tl[:, 3]) >= 0).all()
    assert staged.timeline_read().shape == (0, 4)                                 # read clears the record
    # a device-resident source is computed in place (no staging)
    a, b = StreamEngine(blob, n_streams=13), StreamEngine(blob, n_streams=13)
    assert torch.equal(a.predict_clip_remote(dev.data_ptr(), 9600), b.predict_clip(dev))


def test_host_path_is_ordered_after_reset(torch_cuda):
    """ADVICE r01: reset() runs asynchronously on the caller's stream, predict_clip_host on the library's private
    non-blocking streams -- the host call must still see the reset state (65 536 streams make the memset long enough to race)."""
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    blob = _blob("okay_nabu_synth_int8.mww")
    S = 65536
    base = np.stack([synth_audio(1600, 40 + i) for i in range(16)])
    audio = np.ascontiguousarray(np.tile(base, (S // 16, 1)))
    eng = StreamEngine(blob, n_streams=S)
    first = eng.predict_clip_host(audio).copy()
    side = torch.cuda.Stream()
    for _ in range(3):
        with torch.cuda.stream(side):                 # the reset is queued on a non-default stream
            eng.reset()
        again = eng.predict_clip_host(audio)
        assert np.array_equal(again, first)


def test_reset_by_id_list_host_and_device(torch_cuda):
    """mww_reset(ids) / mww_reset_device_ids: the listed streams restart from fresh state (history = silence) while the rest
    of the handle carries on, in live mode (rotated rings) as well; one batch of launches whatever the list length."""
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    for kind in ("f32", "int8"):
        blob = _blob("okay_nabu_synth_%s.mww" % kind)
        S = 64
        audio = np.stack([synth_audio(480 * 40, 300 + i) for i in range(S)])
        dev = torch.from_numpy(audio).cuda()
        eng, fresh = StreamEngine(blob, n_streams=S), StreamEngine(blob, n_streams=S)
        for i in range(20):                                   # 20 live steps: rings are rotated now
            eng.step(dev[:, 480 * i:480 * (i + 1)].contiguous())
        ids = [3, 17, 40, 63]
        l0 = eng.launch_count
        eng.reset(ids[:2])
        eng.reset(torch.tensor(ids[2:], dtype=torch.int32, device="cuda"))
        assert eng.launch_count - l0 <= 12
        # expected: a freshly created engine (new MicroFrontend + freshly loaded interpreter, audio_utils.py:52 /
        # inference.py:36-39) put on the handle's shared phase (buffered samples all zero, pending-row count)
        d = fresh.state_dict()
        d["frontend_buffered"], d["pending_rows"] = eng.frontend_buffered, eng.pending_rows
        fresh.load_state_dict(d)
        for i in range(20, 40):
            chunk = dev[:, 480 * i:480 * (i + 1)].contiguous()
            got, want = eng.step(chunk), fresh.step(chunk)
            # fp32: the live kernel sums the depthwise taps in physical ring order, and the two handles' rings are rotated
            # differently (20 steps apart), so the summation order -- not the values summed -- differs
            if kind == "int8":
                assert torch.equal(got[ids], want[ids]), (kind, i)
            else:
                assert (got[ids] - want[ids]).abs().max().item() <= F32_TOL, (kind, i)
        st, sf = eng.state_dict(), fresh.state_dict()
        for k in ("carry", "estimate", "nn", "pending"):
            if kind == "int8" or k in ("carry", "estimate"):
                assert np.array_equal(st[k][ids], sf[k][ids]), (kind, k)
            else:
                assert np.abs(st[k][ids] - sf[k][ids]).max() <= 1e-4, (kind, k)
        others = [i for i in range(S) if i not in ids]
        assert not np.array_equal(st["nn"][others], sf["nn"][others])


def test_ingest_buffer_single_rank(torch_cuda, monkeypatch):
    """The multi-GPU ingest path with world size 1 (NCCL): IngestBuffer allocation / IPC export, predict_clip_ingest =
    barrier + (in-place on the ingest rank) compute + gather -- identical to one engine, two consecutive calls."""
    from microwakeword_b200.engine import StreamEngine
    from microwakeword_b200.sharding import IngestBuffer, ShardedEngine
    torch = torch_cuda
    blob = _blob("okay_nabu_synth_int8.mww")
    audio = np.stack([synth_audio(9600, 900 + i) for i in range(13)])
    dist = _single_rank_group(torch)
    try:
        dev = torch.from_numpy(audio).cuda()
        one = StreamEngine(blob, n_streams=13)
        sh = ShardedEngine(blob, 13, 0)
        with IngestBuffer(13, 9600, src=0, device=torch.device("cuda", 0)) as ingest:
            ingest.buffer.copy_(dev)
            for _ in range(2):
                want = one.predict_clip(dev)
                got = sh.predict_clip_ingest(ingest)
                assert got.shape == want.shape and torch.equal(got, want)
            torch.cuda.synchronize()
    finally:
        dist.destroy_process_group()


def test_pinned_host_array_and_numa_binding(torch_cuda):
    from microwakeword_b200.engine import bind_host_thread, host_array
    a = host_array((1024, 480), np.int16, 0)
    a[:] = 7
    assert a.shape == (1024, 480) and a.dtype == np.int16 and int(a.sum()) == 7 * 1024 * 480
    node = a.base.base.numa_node if hasattr(a.base, "base") else None
    t = torch_cuda.from_numpy(a)
    assert t.cuda().sum().item() == 7 * 1024 * 480
    before = os.sched_getaffinity(0)
    got = bind_host_thread(0)
    after = os.sched_getaffinity(0)
    assert after <= before and len(after) >= 1 and (got == -1 or node in (None, got))
    os.sched_setaffinity(0, before)


@pytest.mark.parametrize("step_ms", [20, 10, 30, 7, 25])
def test_tf_op_path_honours_window_step(torch_cuda, step_ms):
    """a3 (audio_utils.py:69-81): use_c=False forwards step_ms to the frontend op; default 20 ms.  Bit-exact against the oracle
    frontend constructed with that step, whole clips and chunked streaming (carry with a hop that is not 10 ms)."""
    from microwakeword.audio.audio_utils import generate_features_for_clip
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    clips = [synth_audio(16000, 60 + step_ms), edge_case_audio(9000)[2], synth_audio(700, 3)]
    for clip in clips:
        fe = oracle.Frontend((16000, 30, step_ms, 40, 125.0, 7500.0))
        fe.reset()
        want = fe.stream(clip)
        got = generate_features_for_clip(clip, step_ms=step_ms, use_c=False)
        assert got.dtype == np.uint16 and got.shape == want.shape and np.array_equal(got, want), (step_ms, clip.size)
    if step_ms == 20:
        assert np.array_equal(generate_features_for_clip(clips[0], use_c=False), want_default(clips[0]))
    # streaming with carried state, many streams (one CTA per stream), odd chunk sizes
    audio = np.stack([synth_audio(12000, 90 + i) for i in range(9)])
    eng = StreamEngine(None, n_streams=9)
    eng.set_window_step(16 * step_ms)
    parts, pos = [], 0
    for n in (5000, 1234, 16, 3000, 2750):
        parts.append(_u16(eng.features(torch.from_numpy(np.ascontiguousarray(audio[:, pos:pos + n])).cuda())))
        pos += n
    got = np.concatenate(parts, 1)
    for i in range(9):
        fe = oracle.Frontend((16000, 30, step_ms, 40, 125.0, 7500.0))
        fe.reset()
        want = fe.stream(audio[i])
        assert got[i].shape == want.shape and np.array_equal(got[i], want), (step_ms, i)
    if eng.frontend_buffered:                # a 30 ms step consumes the 12 000 samples exactly
        with pytest.raises(Exception):
            eng.set_window_step(320)         # samples are buffered
    eng.reset_frontend()
    eng.set_window_step(160)
    with pytest.raises(Exception):
        eng.set_window_step(481)


def want_default(clip):
    fe = oracle.Frontend((16000, 30, 20, 40, 125.0, 7500.0))
    fe.reset()
    return fe.stream(clip)
