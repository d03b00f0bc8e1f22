"""The batched form of the reference's state-carrying evaluation loop (microwakeword_b200.batched,
Model.predict_spectrograms) and the streaming accuracy test of its harness (evaluation.tflite_model_accuracy), on the CPU:
  * the warm-up bound W = stride * warmup_steps(arch) is exact and tight: the oracle run over a sequence of tracks one
    step after another equals the same sequence cut into segments that each start from a zero state fed the W rows before
    them, bit for bit (fp32 and int8), and W - stride rows are not enough;
  * the planner's invariants;
  * the oracle restatement of tflite_model_accuracy / compute_metrics / metrics_to_string, and the product's host
    functions, equal the output of the reference's own functions (tests/golden/accuracy_golden.npz)."""

import functools
import json
import os

import numpy as np
import pytest

import oracle
from conftest import GOLDEN, synth_audio
from microwakeword_b200 import batched, evaluation
from microwakeword_b200 import model_file as MF
from oracle import accuracy_ref as A
from oracle import mixednet_ref as R

ARCHS = {
    "okay_nabu": R.Spec(),
    "one_tap_block": R.Spec(48, 7, 3, (64, 32, 96), ((9,), (3, 5, 7, 9), (1,)), head_rows=3),       # block 2: largest kernel 1
    "k0_equals_stride": R.Spec(8, 4, 4, (16, 16), ((2,), (4,)), head_rows=2),                        # no first-conv ring
}


def _arch(spec):
    return MF.Arch(spec.first_conv_filters, spec.first_conv_kernel_size, spec.stride, spec.pointwise_filters,
                   spec.mixconv_kernel_sizes, spec.head_rows)


def _features(n_rows, seed):
    audio = synth_audio(160 * (n_rows + 2), seed)[None, :]
    feats, _ = oracle.run_pipeline(None, audio, want_probs=False)
    return feats[0, :n_rows]                                          # uint16 [n_rows, 40]


@functools.lru_cache(maxsize=None)
def _models(name):
    spec = ARCHS[name]
    f32 = R.fold_bn(spec, R.init_synthetic(spec, 0))
    calib = _features(600, 7000)
    calib = calib[: calib.shape[0] // spec.stride * spec.stride].reshape(-1, spec.stride, 40)
    q8 = R.quantize_model(f32, calib.astype(np.float32) * R.FEATURE_SCALE)
    return spec, f32, MF.write_container(q8)


@pytest.fixture(scope="module", params=list(ARCHS))
def models(request):
    return _models(request.param)


def _run_f32(f32, rows, model=None):
    m = model or R.FoldedStreamingF32(f32)
    s = m.spec.stride
    x = rows.astype(np.float32) * R.FEATURE_SCALE
    return np.asarray([m.step(x[i:i + s]) for i in range(0, x.shape[0] // s * s, s)], np.float32), m


def _run_i8(blob, rows):
    return oracle.MixedNet(blob).predict_u16(rows)


def _segmented(run, rows, p, stride, warm_steps):
    """Segment i of the plan on its own model: zero state, then the warm_steps steps before the segment (discarded)."""
    out = []
    for i in range(p.n_streams):
        a, b = i * p.seg_steps, min((i + 1) * p.seg_steps, p.total_steps)
        w = 0 if i == 0 else warm_steps
        out.append(run(rows[(a - w) * stride:b * stride])[w:])
    return np.concatenate(out)


def _warmup_case(spec, seed):
    """A random test set long enough for three segments, its plan and its rows."""
    w = batched.warmup_steps(_arch(spec))
    rng = np.random.default_rng(seed)
    steps = rng.integers(0, 3 * w, 40)
    while steps.sum() < 12 * w:
        steps = np.concatenate([steps, rng.integers(1, 3 * w, 4)])
    p = batched.plan(steps, spec.stride, spec.stride * w, max_streams=3)
    assert p.n_streams == 3 and p.seg_steps >= w
    return w, p, _features(p.total_steps * spec.stride, 100 * seed)


def _runs(f32, blob):
    return (("f32", lambda r: _run_f32(f32, r)[0]), ("int8", lambda r: _run_i8(blob, r)))


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_warmup_bound_is_exact_and_tight(models, seed):
    """W rows of warm-up give the sequential output bit for bit (fp32 and int8)."""
    spec, f32, blob = models
    w, p, rows = _warmup_case(spec, seed)
    if spec.first_conv_kernel_size == 5 and spec.stride == 3 and spec.head_rows == 17:
        assert w == 67                                                # okay_nabu: 201 rows
    for kind, run in _runs(f32, blob):
        seq = run(rows)
        assert seq.size == p.total_steps
        assert np.array_equal(_segmented(run, rows, p, spec.stride, w), seq), kind


def test_warmup_bound_is_tight():
    """W - stride rows of warm-up are not enough: for every geometry, fp32 and int8 each differ from the sequential output
    for at least one of the seeds (a ReLU can hide one stale ring row for a particular input)."""
    for name in ARCHS:
        spec, f32, blob = _models(name)
        differs = {"f32": False, "int8": False}
        for seed in (1, 2, 3):
            w, p, rows = _warmup_case(spec, seed)
            for kind, run in _runs(f32, blob):
                differs[kind] |= not np.array_equal(_segmented(run, rows, p, spec.stride, w - 1), run(rows))
        assert differs == {"f32": True, "int8": True}, name


def test_final_state_depends_only_on_the_last_warmup_steps(models):
    """Model.predict_spectrograms leaves the model in the state after the last real row by replaying the last
    warmup_steps steps on it: the state after any history followed by those steps equals the sequential state."""
    spec, f32, _ = models
    w = batched.warmup_steps(_arch(spec))
    rows = _features((3 * w + 5) * spec.stride, 77)
    _, seq = _run_f32(f32, rows)
    _, other = _run_f32(f32, _features(20 * spec.stride, 78))           # a model holding some unrelated earlier state
    _, tail = _run_f32(f32, rows[-w * spec.stride:], other)
    for a, b in [(seq.st_first, tail.st_first), (seq.st_head, tail.st_head)] + list(zip(seq.st_block, tail.st_block)):
        assert np.array_equal(a, b)


# ---------------------------------------------------------------------------------------------------------- planner
def _check_plan(steps, stride, w_rows, cap):
    p = batched.plan(steps, stride, w_rows, cap)
    n = int(np.sum(steps))
    w = -(-w_rows // stride)
    assert p.total_steps == n and p.warmup_steps == w
    assert 1 <= p.n_streams <= cap
    if n == 0:
        return p
    assert p.n_streams == min(max(n // (4 * max(w, 1)), 1), cap) or p.n_streams == -(-n // p.seg_steps)
    assert (p.n_streams - 1) * p.seg_steps < n <= p.n_streams * p.seg_steps           # no empty segment, nothing left over
    assert 1 <= p.last_segment_steps <= p.seg_steps
    if p.n_streams > 1:
        assert p.seg_steps >= w and p.seg_steps * stride >= w_rows                    # L >= W
        assert p.n_streams * w <= n // 4 + w                                            # warm-up is a bounded share
    # offsets cover every step exactly once, in track order
    cover = np.zeros(p.n_streams * p.seg_steps, np.int32)
    for o, k in zip(p.track_offsets, steps):
        cover[o:o + k] += 1
    assert (cover[:n] == 1).all() and (cover[n:] == 0).all()
    return p


@pytest.mark.parametrize("stride,w_rows", [(3, 201), (1, 12), (4, 12), (2, 7)])
def test_planner_invariants(stride, w_rows):
    rng = np.random.default_rng(stride * 100 + w_rows)
    w = -(-w_rows // stride)
    cases = [[], [0], [0, 1, 2, 3], [1] * 5, [3, 0, 2, 1] * 50, [int(v) for v in rng.integers(0, 50, 300)],
             [10 * 4 * w * 7 + 3],                                      # one track spanning several segments
             [4 * w - 1], [4 * w], [8 * w - 1], [8 * w], [5, 40 * w, 0, 2 * w, 1]]
    for steps in cases:
        for cap in (1, 2, 3, 65536):
            p = _check_plan(np.asarray(steps, np.int64), stride, w_rows, cap)
            if sum(steps) and sum(steps) < 4 * w:
                assert p.n_streams == 1                                  # too little work to be worth a warm-up
    assert batched.plan([4 * w * 100], stride, w_rows, 65536).n_streams == 100
    assert batched.plan([4 * w * 100], stride, w_rows, 16).n_streams == 16
    with pytest.raises(ValueError):
        batched.plan([-1], stride, w_rows)


def test_packed_tracks_move_to_the_requested_device():
    """Probabilities left on the model's GPU are brought to the device the detection kernels run on."""
    import torch
    from microwakeword_b200 import detection
    packed = detection._Packed(torch.arange(6, dtype=torch.float32), [0, 2], [2, 4])
    flat, offs, lens_d, lens = detection._pack(packed, torch.device("meta"))
    assert flat.device.type == offs.device.type == lens_d.device.type == "meta"
    assert flat.shape == (6,) and list(lens) == [2, 4] and len(packed) == 2


def test_planner_on_the_roc_test_set():
    """okay_nabu, three ambient tracks and five positive clips of tests/test_detection.py: 888 steps -> S = 3."""
    steps = [600 // 3, 697 // 3, 350 // 3] + [204 // 3] * 5
    p = _check_plan(np.asarray(steps), 3, 201, 65536)
    assert p.n_streams == 3 and p.seg_steps == 296


# ---------------------------------------------------------------------------------------------------------- accuracy
@pytest.fixture(scope="module")
def acc_gold():
    g = np.load(os.path.join(GOLDEN, "accuracy_golden.npz"))
    split = lambda flat, lengths: [list(flat[a:a + n]) for a, n in zip(np.concatenate([[0], np.cumsum(lengths)[:-1]]), lengths)]
    return dict(clips=split(g["clip_probs"], g["clip_lengths"]), truth=[bool(v) for v in g["clip_truth"]],
                amb=split(g["amb_probs"], g["amb_lengths"]), duration_s=float(g["duration_s"]),
                cases=json.loads(str(g["cases"])), direct=json.loads(str(g["direct"])))


def _same_metrics(a, b):
    assert set(a) == set(b)
    for k in a:
        assert (np.isnan(a[k]) and np.isnan(b[k])) or a[k] == b[k], (k, a[k], b[k])


def test_accuracy_oracle_equals_reference_output(acc_gold):
    g = acc_gold
    for c in g["cases"]:
        ambient = c["data_set"].endswith("ambient")
        tracks = g["amb"] if ambient else g["clips"]
        truth = [False] * len(tracks) if ambient else g["truth"]
        m, text = A.tflite_model_accuracy(tracks, truth, ambient, c["min_gap"], g["duration_s"])
        _same_metrics(m, c["metrics"])
        assert text == c["text"]
    for d in g["direct"]:
        for impl in (A, evaluation):
            m = impl.compute_metrics(*d["args"])
            _same_metrics(m, d["metrics"])
            assert impl.metrics_to_string(m) == d["text"]


def test_accuracy_rule_small_cases():
    assert A.accuracy_track([0.6, 0.4, 0.6], 0) == (1, True)          # index 0: 0 - 0 > 0 fails; index 2 counts
    assert A.accuracy_track([0.4, 0.6, 0.4, 0.6], 1) == (1, True)     # index 1: 1 - 0 > 1 fails; index 3 counts
    assert A.accuracy_track([0.4, 0.6, 0.4, 0.6], 3) == (0, True)     # both crossings within the first 3 steps
    assert A.accuracy_track([0.5, 0.5], 0) == (0, False)             # strictly above 0.5
    assert A.accuracy_track([], 0) == (0, None)
    with pytest.raises(IndexError):
        A.tflite_model_accuracy([[0.9], []], [True, True], False, 0)
