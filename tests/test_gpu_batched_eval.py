"""GPU side of the batched state-carrying evaluation pass (Model.predict_spectrograms, microwakeword_b200.batched), of
mww_copy_nn_state, and of the streaming accuracy test (mww_accuracy_counts, evaluation.tflite_model_accuracy).  The
warm-up bound and the planner are checked on the CPU in tests/test_batched_eval.py."""

import json
import os

import numpy as np
import pytest

import oracle
from conftest import GOLDEN, synth_audio
from microwakeword_b200 import _lib, batched, detection, evaluation
from microwakeword_b200 import model_file as MF
from microwakeword_b200.inference import Model
from oracle import accuracy_ref as A
from oracle import mixednet_ref as R

pytestmark = pytest.mark.gpu

GENERIC = R.Spec(48, 7, 3, (64, 32, 96), ((9,), (3, 5, 7, 9), (1,)), head_rows=3)


def _feats(n_rows, seed):
    audio = synth_audio(160 * (n_rows + 2), seed)[None, :]
    return oracle.run_pipeline(None, audio, want_probs=False)[0][0, :n_rows]


def _generic_blob(kind):
    f32 = R.fold_bn(GENERIC, R.init_synthetic(GENERIC, 0))
    if kind == "f32":
        return MF.write_container(f32)
    calib = _feats(600, 7000)
    calib = calib[: calib.shape[0] // GENERIC.stride * GENERIC.stride].reshape(-1, GENERIC.stride, 40)
    return MF.write_container(R.quantize_model(f32, calib.astype(np.float32) * R.FEATURE_SCALE))


def _blob(model, kind):
    if model == "okay_nabu":
        return open(os.path.join(GOLDEN, "okay_nabu_synth_%s.mww" % kind), "rb").read()
    return _generic_blob(kind)


def _tracks(rows, rng, n_tracks):
    """Ragged tracks cut from a feature sequence: 0..5 rows, clip-sized ones and a few long ones."""
    out, at = [], 0
    for i in range(n_tracks):
        n = int(rng.integers(0, 6)) if i % 3 == 0 else (int(rng.integers(150, 260)) if i % 7 else int(rng.integers(600, 1500)))
        out.append(rows[at % (rows.shape[0] - n):at % (rows.shape[0] - n) + n])
        at += n
    return out


@pytest.mark.parametrize("model", ["okay_nabu", "generic"])
@pytest.mark.parametrize("kind", ["int8", "f32"])
@pytest.mark.parametrize("rows", ["u16", "f32", "i8", "mixed"])
def test_predict_spectrograms_equals_the_loop(torch_cuda, model, kind, rows):
    if rows == "i8" and kind != "int8":
        pytest.skip("pre-quantised rows exist for int8 models only")
    blob = _blob(model, kind)
    rng = np.random.default_rng(sum(map(ord, model + kind + rows)))
    feats = _feats(6000, 31)
    loop, batch = Model(blob), Model(blob)
    tracks = _tracks(feats, rng, 60)
    if rows == "f32":
        tracks = [t.astype(np.float32) * R.FEATURE_SCALE for t in tracks]
    elif rows == "i8":
        tracks = [R.quantize_input(t.astype(np.float32) * R.FEATURE_SCALE, loop.input_details[0]["quantization"][0],
                                   loop.input_details[0]["quantization"][1]) for t in tracks]
    elif rows == "mixed":
        tracks = [t.astype(np.float64) * R.FEATURE_SCALE if i % 2 else t for i, t in enumerate(tracks)]
    for m in (loop, batch):                                           # a non-zero starting state
        m.predict_spectrogram(feats[:300])
        m.predict_spectrogram(feats[500:530])
    steps = [t.shape[0] // loop.input_feature_slices for t in tracks]
    p = batched.plan(steps, loop.input_feature_slices, loop.input_feature_slices * batched.warmup_steps(loop._arch()), 65536)
    ends = p.track_offsets + np.asarray(steps) - 1
    assert p.n_streams > 2 and ((p.track_offsets // p.seg_steps) != (ends // p.seg_steps))[np.asarray(steps) > 0].sum() >= 2
    want = [loop.predict_spectrogram(t) for t in tracks]
    got = batch.predict_spectrograms(tracks)
    assert [len(g) for g in got] == [len(w) for w in want]
    assert all(type(v) is np.float32 for g in got for v in g) and all(type(g) is list for g in got)
    flat_g, flat_w = np.concatenate([np.asarray(g, np.float32) for g in got]), np.concatenate([np.asarray(w, np.float32) for w in want])
    s_got, s_want = batch.engine.state_dict(), loop.engine.state_dict()
    assert s_got["pending_rows"] == s_want["pending_rows"] == 0
    after_g, after_w = batch.predict_spectrogram(feats[1000:1300]), loop.predict_spectrogram(feats[1000:1300])
    if kind == "int8":
        assert np.array_equal(flat_g, flat_w)
        assert np.array_equal(s_got["nn"], s_want["nn"])
        assert np.array_equal(after_g, after_w)
    else:
        assert np.abs(flat_g - flat_w).max() <= 1e-5
        assert np.abs(s_got["nn"] - s_want["nn"]).max() <= 1e-4
        assert np.abs(np.asarray(after_g) - np.asarray(after_w)).max() <= 1e-5
    assert 0.01 < flat_w.mean() < 0.99 and flat_w.std() > 1e-3         # the comparison is not vacuous


def test_predict_spectrograms_other_chunk_stride_and_edges(torch_cuda):
    blob = _blob("okay_nabu", "int8")
    feats = _feats(4000, 5)
    tracks = [feats[:0], feats[:1], feats[:2], feats[3:6], feats[10:2300], feats[100:1900]]
    loop, batch = Model(blob, stride=2), Model(blob, stride=2)          # chunks overlap (inference.py:98-105)
    want = [loop.predict_spectrogram(t) for t in tracks]
    assert batch.predict_spectrograms(tracks) == want
    assert np.array_equal(batch.engine.state_dict()["nn"], loop.engine.state_dict()["nn"])
    assert batch.predict_spectrograms([]) == [] and batch.predict_spectrograms([feats[:1]]) == [[]]
    batch.release_batched()                                           # frees the kept buffers; the next call allocates them again
    assert batch.predict_spectrograms(tracks[4:]) == [loop.predict_spectrogram(t) for t in tracks[4:]]
    q = Model(blob)
    with pytest.raises(ValueError):
        q.predict_spectrograms([feats[:30], np.zeros((30, 40), np.int8)])
    q.engine.infer(torch_cuda.zeros((1, 1, 40), dtype=torch_cuda.float32, device="cuda"))
    with pytest.raises(RuntimeError):                                  # pending rows from a partial step
        q.predict_spectrograms([feats[:30]])
    with pytest.raises(ValueError):
        Model(blob, batch=2).predict_spectrograms([feats[:30]])


def test_predict_spectrograms_at_scale(torch_cuda):
    """>= 16 384 streams (past the first wave of the persistent grids): sampled segments against the int8 oracle run from a
    zero state over [segment start - W, segment end)."""
    blob = _blob("okay_nabu", "int8")
    w = 67
    s_min = 16384
    n_steps = (s_min + 100) * 4 * w + 123                           # the plan lowers S to ceil(N / L): leave a margin
    rng = np.random.default_rng(7)
    base = _feats(3 * 4000, 11)
    rows = base[rng.integers(0, base.shape[0] - 600, n_steps * 3 // 600 + 1)[:, None] + np.arange(600)[None, :]].reshape(-1, 40)
    rows = rows[:n_steps * 3]
    cuts = np.sort(rng.choice(np.arange(1, n_steps), 499, replace=False)) * 3
    tracks = np.split(rows, cuts)
    m = Model(blob)
    flat, offsets, lengths = m._predict_spectrograms_device(tracks)
    p = batched.plan(lengths, 3, 3 * w, 65536)
    assert p.n_streams >= s_min and int(lengths.sum()) == n_steps
    flat = flat.cpu().numpy()
    ref = oracle.MixedNet(blob)
    sample = sorted(set([0, p.n_streams - 1] + [int(v) for v in rng.integers(1, p.n_streams - 1, 220)]))
    assert len(sample) >= 200
    for i in sample:
        a, b = i * p.seg_steps, min((i + 1) * p.seg_steps, n_steps)
        warm = min(w, a)
        ref.reset()
        want = ref.predict_u16(rows[(a - warm) * 3:b * 3])[warm:]
        assert np.array_equal(flat[a:b], want), i


# ------------------------------------------------------------------------------------------------ mww_copy_nn_state
def test_copy_nn_state(torch_cuda):
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    blob = _blob("okay_nabu", "int8")
    feats = torch.from_numpy(_feats(400, 3).astype(np.float32) * R.FEATURE_SCALE).cuda()
    rows = lambda n_streams, start, n: torch.stack([feats[start + 7 * i:start + 7 * i + n] for i in range(n_streams)]).contiguous()
    a, b = StreamEngine(blob, n_streams=4), StreamEngine(blob, n_streams=3)
    a.infer(rows(4, 0, 240))
    audio = torch.from_numpy(np.stack([synth_audio(900, 40 + i) for i in range(3)])).cuda()
    b.predict_clip(audio)                                             # 3 rows: a whole step, 420 samples left in the carry
    b.infer(rows(3, 10, 60))
    fe_before = b.state_dict()
    before = fe_before["nn"]
    assert b.frontend_buffered == 420 and fe_before["carry"].any() and fe_before["estimate"].any()
    for i in range(5):                                                # live calls: a's rings are left rotated
        a.infer(rows(4, 240 + 3 * i, 3))
    b.copy_nn_state([2, 0], a, [1, 3])
    src = a.state_dict()["nn"]
    got = b.state_dict()["nn"]
    assert np.array_equal(got[2], src[1]) and np.array_equal(got[0], src[3]) and np.array_equal(got[1], before[1])
    assert not np.array_equal(src[1], src[3]) and not np.array_equal(got[1], got[2])
    a.copy_nn_state([0], b, [1])                                      # and back: a round trip is exact
    assert np.array_equal(a.state_dict()["nn"][0], before[1])
    a.copy_nn_state([1, 2], a, [0, 0])                                # dst == src
    assert np.array_equal(a.state_dict()["nn"][2], before[1])
    fe_after = b.state_dict()                                         # frontend state is not touched
    assert np.array_equal(fe_after["carry"], fe_before["carry"]) and np.array_equal(fe_after["estimate"], fe_before["estimate"])
    assert fe_after["frontend_buffered"] == 420
    other = StreamEngine(_blob("okay_nabu", "f32"), n_streams=3)
    t = MF.read_container(blob)                                       # same geometry and dtype, other weights: only the model hash differs
    t["q/head/bias"] = np.asarray(t["q/head/bias"]) + 1
    twin = StreamEngine(MF.write_container(t), n_streams=3)
    assert twin.is_quantized and twin.state_elements == b.state_elements
    for call in (lambda: b.copy_nn_state([0], other, [0]), lambda: b.copy_nn_state([0], twin, [0]), lambda: b.copy_nn_state([3], a, [0]), lambda: b.copy_nn_state([0], a, [4]),
                 lambda: b.copy_nn_state([-1], a, [0])):
        with pytest.raises(_lib.MwwError) as e:
            call()
        assert e.value.code == -1
    a.infer(rows(4, 0, 1))                                            # a pending row
    with pytest.raises(_lib.MwwError) as e:
        b.copy_nn_state([0], a, [0])
    assert e.value.code == -1 and "pending" in str(e.value)


# ------------------------------------------------------------------------------------------------ accuracy
def test_accuracy_kernel_equals_oracle_on_golden_tracks(torch_cuda):
    g = np.load(os.path.join(GOLDEN, "accuracy_golden.npz"))
    for probs, lengths in ((g["clip_probs"], g["clip_lengths"]), (g["amb_probs"], g["amb_lengths"])):
        offs = np.concatenate([[0], np.cumsum(lengths)[:-1]])
        tracks = [probs[a:a + n] for a, n in zip(offs, lengths)]
        for gap in (0, 3, 20):
            fa, last = detection.accuracy_counts(tracks, gap)
            want = [A.accuracy_track(t, gap) for t in tracks]
            assert list(fa) == [c for c, _ in want]
            assert list(last) == [bool(v) for _, v in want]
    # and the cases the golden pins end to end, through the metric bookkeeping
    for c in json.loads(str(g["cases"])):
        ambient = c["data_set"].endswith("ambient")
        lengths, probs = (g["amb_lengths"], g["amb_probs"]) if ambient else (g["clip_lengths"], g["clip_probs"])
        offs = np.concatenate([[0], np.cumsum(lengths)[:-1]])
        fa, last = detection.accuracy_counts([probs[a:a + n] for a, n in zip(offs, lengths)], c["min_gap"])
        truth = g["clip_truth"]
        if ambient:
            text = "false accepts = {}; false accepts per hour = {:.4}".format(float(fa.sum()), float(fa.sum()) / (float(g["duration_s"]) / 3600.0))
        else:
            hit, pos = truth == last, truth
            m = evaluation.compute_metrics(float((hit & pos).sum()), float((hit & ~pos).sum()), float((~hit & ~pos).sum()), float((~hit & pos).sum()))
            text = evaluation.metrics_to_string(m)
        assert text == c["text"]


@pytest.mark.parametrize("ambient", [False, True])
def test_tflite_model_accuracy_equals_oracle_composition(torch_cuda, ambient):
    """test.py:406-517 end to end (int8 okay_nabu: exact): Model -> batched pass -> accuracy kernel -> metrics, against one
    oracle interpreter fed the same float32 fingerprints in order, then the oracle restatement of the metric rule."""
    path = os.path.join(GOLDEN, "okay_nabu_synth_int8.mww")
    blob = open(path, "rb").read()
    feats = _feats(9000, 17)
    rng = np.random.default_rng(3)
    if ambient:
        fps = [feats[a:a + n] for a, n in ((0, 3000), (2000, 2900), (100, 7), (5000, 3999))]
    else:
        fps = [feats[s:s + 204] for s in rng.integers(0, 8700, 120)]
    raw = [f[:f.shape[0] // 3 * 3] if ambient else f for f in fps]
    fps = [f.astype(np.float32) * R.FEATURE_SCALE for f in fps]        # the reference's get_data gives scaled features (exact)
    truth = rng.random(len(fps)) < 0.5
    got_m, got_s = evaluation.tflite_model_accuracy(Model(path), fps, truth, ambient, 5, ambient_duration_s=123.0)
    class LoopOnly:                                                   # an object with nothing but predict_spectrogram
        def __init__(self, m):
            self.predict_spectrogram = m.predict_spectrogram
    assert evaluation.tflite_model_accuracy(LoopOnly(Model(path)), fps, truth, ambient, 5, ambient_duration_s=123.0)[1] == got_s
    ref = oracle.MixedNet(blob)                                       # one interpreter, never reset (inference.py:52-64)
    probs = [list(ref.predict_u16(u)) for u in raw]
    want_m, want_s = A.tflite_model_accuracy(probs, truth, ambient, 5, 123.0)
    assert got_s == want_s
    for k in want_m:
        assert (np.isnan(want_m[k]) and np.isnan(got_m[k])) or got_m[k] == want_m[k], k
    if ambient:
        assert want_m["count"] > 0
    else:
        assert 0 < want_m["accuracy"] < 1
