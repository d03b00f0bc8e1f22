"""GPU side of hybrid models (microwakeword_b200/csrc/mww_nn_generic.cu, nn_generic_hybrid_kernel): the float streaming
.tflite whose large conv / depthwise / dense weights are per-channel int8 (dynamic-range quantisation), through every
entry point a float model has, against the hybrid oracle (tests/hybrid_ref, [UPSTREAM-RECALL]).  NN rings are bit-identical to the
oracle's after every call; probabilities agree within 1e-6 (only the final sigmoid's expf may differ).  The phase functions
are checked on the CPU in tests/test_hybrid.py."""

import os

import numpy as np
import pytest

import oracle
import hybrid_ref as HR
import tflite_hybrid_writer as HW
import tflite_writer as TW
from conftest import GOLDEN, synth_audio
from microwakeword_b200 import detection, evaluation
from microwakeword_b200 import model_file as MF
from microwakeword_b200 import tflite_file as TF
from oracle import mixednet_ref as R

pytestmark = pytest.mark.gpu

PROB_TOL = 1e-6


def converter_rule(op, n):
    return n >= 1024


def all_rule(op, n):
    return True


GEOMS = {
    "okay_nabu": (R.Spec(), converter_rule, True),
    "stride2_three_groups": (R.Spec(16, 6, 2, (40,), ((7, 11, 13),), head_rows=9), all_rule, False),
    "split_threshold": (R.Spec(64, 5, 3, (32, 48), ((9, 33), (3,)), head_rows=5), converter_rule, True),
}


def _tflite(name):
    spec, rule, fc_asym = GEOMS[name]
    if name == "okay_nabu":
        f32 = MF.load(os.path.join(GOLDEN, "okay_nabu_synth_f32.mww"))
    else:
        f32 = R.fold_bn(spec, R.init_synthetic(spec, 0))
    return HW.write_hybrid_mixednet(f32, rule, fc_asym)


def _container(name):
    return MF.write_container(TF.tensors_from_tflite(_tflite(name)))


class OracleStreams:
    """One oracle interpreter per stream, fed float rows with its own pending-row buffer (what the engine keeps per stream)"""

    def __init__(self, blob, n):
        self.m = [HR.HybridNet(blob) for _ in range(n)]
        self.stride = self.m[0].stride
        self.pend = [np.zeros((0, 40), np.float32) for _ in range(n)]

    def feed(self, k, rows_f32):
        buf = np.concatenate([self.pend[k], rows_f32])
        s = self.stride
        out = [self.m[k].step(buf[j:j + s])[0] for j in range(0, buf.shape[0] // s * s, s)]
        self.pend[k] = buf[buf.shape[0] // s * s:]
        return np.asarray(out, np.float32)


def _check_state(eng, ref, streams):
    sd = eng.state_dict()
    for k, s in enumerate(streams):
        assert np.array_equal(sd["nn"][s], ref.m[k].state()), s
        n = ref.pend[k].shape[0]
        assert sd["pending_rows"] == n
        if n:
            assert np.array_equal(sd["pending"][s, :n], ref.pend[k])


def test_hybrid_okay_nabu_never_reaches_the_compiled_in_kernels(torch_cuda):
    """same weights as a pure-float .tflite: today's fp32 results (the compiled-in kernels, fp32 tolerance); as a hybrid
    .tflite: the oracle's hybrid arithmetic -- the path is chosen by the file's content"""
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    hy = TF.tensors_from_tflite(_tflite("okay_nabu"))
    plain = {k: v for k, v in hy.items() if not k.startswith("hy/")}          # the dequantised weights as float32
    audio = np.stack([synth_audio(16000, 2100 + i) for i in range(8)])
    dev = torch.from_numpy(audio).cuda()
    for tensors, kind in ((plain, "f32"), (hy, "hybrid")):
        blob = MF.write_container(tensors)
        tfl = _tflite("okay_nabu") if kind == "hybrid" else TW.write_streaming_mixednet(plain)
        if kind == "hybrid":
            _, want = HR.run_pipeline(blob, audio, threads=4)
        else:
            _, want = oracle.run_pipeline(blob, audio, want_features=False, threads=4)
        for model in (blob, tfl):
            eng = StreamEngine(model, n_streams=8)
            assert not eng.is_quantized
            got = eng.predict_clip(dev).cpu().numpy()
            assert got.shape == want.shape
            assert np.abs(got - want).max() <= (PROB_TOL if kind == "hybrid" else 1e-5), kind
    _, p_plain = oracle.run_pipeline(MF.write_container(plain), audio, want_features=False, threads=4)
    _, p_hy = HR.run_pipeline(MF.write_container(hy), audio, threads=4)
    assert not np.array_equal(p_plain, p_hy)


@pytest.mark.parametrize("audio_dtype", ["int16", "float32"])
def test_clip_at_65536_streams(torch_cuda, audio_dtype):
    """65 536 streams x a 3 s predict_clip on hybrid okay_nabu; 96 streams spread over the grid (first, last, and every
    persistent wave) are checked against the oracle: probabilities within 1e-6, rings bit-identical."""
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    S, N = 65536, 48000
    blob = _container("okay_nabu")
    g = torch.Generator(device="cuda").manual_seed(7)
    base = torch.from_numpy(np.stack([synth_audio(N, 3000 + i) for i in range(64)])).cuda()
    audio = base.repeat(S // 64, 1)                                  # 64 clips, each stream with its own added noise
    for a in range(0, S, 4096):
        noisy = audio[a:a + 4096].to(torch.int32) + torch.randint(-300, 300, (4096, N), device="cuda", generator=g, dtype=torch.int32)
        audio[a:a + 4096] = noisy.clamp(-32768, 32767).to(torch.int16)
    del noisy
    eng = StreamEngine(blob, n_streams=S)
    src = audio if audio_dtype == "int16" else audio.to(torch.float32) / 32768.0
    got = eng.predict_clip(src).cpu().numpy()
    sample = np.unique(np.concatenate([[0, 1, S - 1, S - 2], np.linspace(0, S - 1, 92).astype(np.int64)]))
    a_host = audio[torch.from_numpy(sample).cuda()].cpu().numpy()
    del src, audio
    torch.cuda.empty_cache()
    feats, want = HR.run_pipeline(blob, a_host, threads=8)
    assert got.shape == (S, want.shape[1])
    assert np.abs(got[sample] - want).max() <= PROB_TOL
    assert want.std() > 1e-3
    nn = eng.state_dict()["nn"]
    for k, s in enumerate(sample):
        m = HR.HybridNet(blob)
        m.predict_u16(feats[k])
        assert np.array_equal(nn[s], m.state()), s


@pytest.mark.parametrize("name", list(GEOMS))
def test_ragged_calls_over_several_waves(torch_cuda, name):
    """6 x SMs + 37 streams through calls of 1 .. 257 steps, entering with 0, 1 and 2 pending rows, uint16 and float32 rows:
    rings and pending rows bit-identical to the oracle after every call"""
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    blob = _container(name)
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    S = 6 * sm + 37
    eng = StreamEngine(blob, n_streams=S)
    s = eng.stride
    check = np.unique(np.asarray([0, 1, sm - 1, sm, 3 * sm + 5, S - 2, S - 1]))
    ref = OracleStreams(blob, len(check))
    rng = np.random.default_rng(11)
    calls = [1, 1, s * 1 - 1, s * 257 + 1, 2, s * 3, s * 40 + 2, s - 1, s * 100, s * 1]
    for i, n in enumerate(calls):
        rows = rng.integers(0, 900, (S, n, 40)).astype(np.uint16)
        rows_f = rows.astype(np.float32) * np.float32(R.FEATURE_SCALE)
        dev = torch.from_numpy(rows_f if i % 2 else rows).cuda()
        got = eng.infer(dev).cpu().numpy()
        for k, st in enumerate(check):
            want = ref.feed(k, rows_f[st])
            assert got.shape[1] == want.size
            assert np.abs(got[st] - want).max(initial=0) <= PROB_TOL, (i, st)
        _check_state(eng, ref, check)


@pytest.mark.parametrize("name", ["okay_nabu", "split_threshold"])
def test_live_steps_reset_state_roundtrip_and_copy(torch_cuda, name):
    """480-sample step() calls, reset(ids), load_state_dict round trips and copy_nn_state"""
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    blob = _container(name)
    S = 24
    audio = np.stack([synth_audio(16000, 4000 + i) for i in range(S)])
    dev = torch.from_numpy(audio).cuda()
    feats, want = HR.run_pipeline(blob, audio, threads=4)
    eng = StreamEngine(blob, n_streams=S)
    parts = [eng.step(dev[:, a:a + 480].contiguous()) for a in range(0, 16000 - 479, 480)]
    live = torch.cat(parts, 1).cpu().numpy()
    assert np.abs(live - want[:, :live.shape[1]]).max() <= PROB_TOL
    ref = OracleStreams(blob, S)
    rows_seen = live.shape[1] * eng.stride + eng.pending_rows
    for k in range(S):
        ref.feed(k, feats[k, :rows_seen].astype(np.float32) * np.float32(R.FEATURE_SCALE))
    _check_state(eng, ref, range(S))
    # load_state_dict round trip: a second engine continues identically
    sd = eng.state_dict()
    twin = StreamEngine(blob, n_streams=S)
    twin.load_state_dict(sd)
    assert np.array_equal(twin.state_dict()["nn"], sd["nn"])
    more = torch.from_numpy(np.stack([synth_audio(4800, 5000 + i) for i in range(S)])).cuda()
    a, b = eng.step(more).cpu().numpy(), twin.step(more).cpu().numpy()
    assert np.array_equal(a, b) and np.array_equal(eng.state_dict()["nn"], twin.state_dict()["nn"])
    # reset(ids): those streams start over like a fresh engine, the others are untouched
    before = eng.state_dict()["nn"]
    eng.reset(stream_ids=[1, 5])
    after = eng.state_dict()["nn"]
    fresh = StreamEngine(blob, n_streams=S).state_dict()["nn"]
    assert np.array_equal(after[[1, 5]], fresh[[1, 5]]) and np.array_equal(np.delete(after, [1, 5], 0), np.delete(before, [1, 5], 0))
    eng.reset()
    ref = OracleStreams(blob, S)
    p = eng.infer(torch.from_numpy(feats[:, :60].copy()).cuda()).cpu().numpy()
    for k in range(S):
        assert np.abs(p[k] - ref.feed(k, feats[k, :60].astype(np.float32) * np.float32(R.FEATURE_SCALE))).max() <= PROB_TOL
    _check_state(eng, ref, range(S))
    # copy_nn_state: stream 3 of a fresh engine takes stream 7 of eng
    dst = StreamEngine(blob, n_streams=S)
    dst.copy_nn_state([3], eng, [7])
    assert np.array_equal(dst.state_dict()["nn"][3], ref.m[7].state())


def test_predict_spectrograms_roc_and_accuracy_on_the_hybrid_tflite(torch_cuda, tmp_path):
    """predict_spectrograms equals the per-track loop bit for bit, state included; streaming_model_roc on the .tflite equals
    the oracle loop's; tflite_model_accuracy runs on it; input / output details are a float model's"""
    from microwakeword_b200.inference import Model
    path = str(tmp_path / "stream_state_internal.tflite")
    with open(path, "wb") as f:
        f.write(_tflite("okay_nabu"))
    blob = _container("okay_nabu")
    audio = synth_audio(160 * 9002, 77)[None, :]
    feats = oracle.run_pipeline(None, audio, want_probs=False)[0][0, :9000]
    rng = np.random.default_rng(4)
    tracks = []
    at = 0
    for i in range(40):
        n = int(rng.integers(0, 6)) if i % 4 == 0 else int(rng.integers(150, 700))
        tracks.append(feats[at % (9000 - n):at % (9000 - n) + n])
        at += n
    loop, batch = Model(path), Model(path)
    assert loop.input_details[0]["dtype"] == np.float32 and loop.output_details[0]["dtype"] == np.float32
    assert not loop.is_quantized_model
    for m in (loop, batch):
        m.predict_spectrogram(feats[:300])
    want = [loop.predict_spectrogram(t) for t in tracks]
    got = batch.predict_spectrograms(tracks)
    assert got == want
    assert np.array_equal(batch.engine.state_dict()["nn"], loop.engine.state_dict()["nn"])

    class OracleLoop:                                                 # the reference's loop on the oracle interpreter
        def __init__(self):
            self.m = HR.HybridNet(blob)

        def predict_spectrogram(self, spec):
            return list(self.m.predict_u16(np.asarray(spec)))

    amb, pos = tracks[:20], tracks[20:]
    r_gpu = detection.streaming_model_roc(Model(path), amb, pos)
    r_ref = detection.streaming_model_roc(OracleLoop(), amb, pos)
    assert r_gpu["auc"] == r_ref["auc"] and np.array_equal(r_gpu["faph"], r_ref["faph"]) and np.array_equal(r_gpu["frr"], r_ref["frr"])
    fps = [feats[s:s + 204].astype(np.float32) * R.FEATURE_SCALE for s in rng.integers(0, 8700, 60)]
    truth = rng.random(len(fps)) < 0.5

    class LoopOnly:
        def __init__(self, m):
            self.predict_spectrogram = m.predict_spectrogram

    got_m, got_s = evaluation.tflite_model_accuracy(Model(path), fps, truth, False, 5)
    assert evaluation.tflite_model_accuracy(LoopOnly(Model(path)), fps, truth, False, 5)[1] == got_s
    assert 0 <= got_m["accuracy"] <= 1
    # predict_clip and predict_nonstreaming accept the file like any float model
    m = Model(path)
    clip = m.predict_clip(synth_audio(16000, 9))
    assert len(clip) > 10 and all(0.0 <= p <= 1.0 for p in clip)
    x = np.stack([feats[i:i + m.nonstreaming_length()] for i in range(0, 400, 100)]).astype(np.float32) * R.FEATURE_SCALE
    assert m.predict_nonstreaming(x).shape[0] == x.shape[0]
