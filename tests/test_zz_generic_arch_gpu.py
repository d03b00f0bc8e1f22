"""GPU side of the run-time-geometry MixedNet path (microwakeword_b200/csrc/mww_nn_generic.cu): models whose architecture
differs from the compiled-in okay_nabu one, through the C-ABI (mww_create -> mww_infer_features / mww_predict_clip /
mww_get_state), against the oracle.  The same phase functions are checked on the CPU in tests/test_generic_arch.py."""

import os

import numpy as np
import pytest

import oracle
from conftest import synth_audio
from microwakeword_b200 import model_file as MF
from oracle import mixednet_ref as R

pytestmark = pytest.mark.gpu

ARCHS = {
    "stride1_two_blocks": R.Spec(24, 3, 1, (32, 48), ((3,), (5, 9)), head_rows=5),
    "stride2_three_groups": R.Spec(16, 6, 2, (40,), ((7, 11, 13),), head_rows=9),
    "wide_first_conv": R.Spec(48, 7, 3, (64, 32, 96), ((9,), (3, 5, 7, 9), (1,)), head_rows=3),
}


def _models(spec):
    f32 = R.fold_bn(spec, R.init_synthetic(spec, 0))
    calib_audio = np.stack([synth_audio(16000, 7000 + i) for i in range(2)])
    calib, _ = oracle.run_pipeline(None, calib_audio, want_probs=False)
    calib = calib.reshape(-1, 40)
    calib = calib[: calib.shape[0] // spec.stride * spec.stride].reshape(-1, spec.stride, 40)
    return f32, R.quantize_model(f32, calib.astype(np.float32) * R.FEATURE_SCALE)


@pytest.mark.parametrize("name", list(ARCHS))
@pytest.mark.parametrize("kind", ["f32", "int8"])
def test_generic_architecture_through_the_c_abi(torch_cuda, name, kind):
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    spec = ARCHS[name]
    f32, q8 = _models(spec)
    blob = MF.write_container(f32 if kind == "f32" else q8)
    audio = np.stack([synth_audio(24000, 1200 + i) for i in range(9)])
    _, want = oracle.run_pipeline(blob, audio, want_features=False, threads=4)
    eng = StreamEngine(blob, n_streams=9)
    assert eng.stride == spec.stride
    dev = torch.from_numpy(audio).cuda()
    got = eng.predict_clip(dev).cpu().numpy()
    assert got.shape == want.shape
    assert np.array_equal(got, want) if kind == "int8" else np.abs(got - want).max() <= 1e-5
    # the same audio in uneven chunks: frontend carry, pending rows and the rings persist across calls
    eng.reset()
    parts = [eng.step(dev[:, a:b].contiguous()) for a, b in ((0, 1000), (1000, 1480), (1480, 9000), (9000, 24000))]
    chunked = torch.cat(parts, 1).cpu().numpy()
    assert chunked.shape == want.shape
    assert np.array_equal(chunked, want) if kind == "int8" else np.abs(chunked - want).max() <= 1e-5
    # feature rows of every dtype through mww_infer_features
    feats, _ = oracle.run_pipeline(None, audio, want_probs=False)
    usable = feats.shape[1] // spec.stride * spec.stride
    eng.reset()
    rows = torch.from_numpy((feats[:, :usable].astype(np.float32) * R.FEATURE_SCALE)).cuda()
    p = eng.infer(rows).cpu().numpy()
    assert np.array_equal(p, want[:, :p.shape[1]]) if kind == "int8" else np.abs(p - want[:, :p.shape[1]]).max() <= 1e-5


def test_generic_state_roundtrip_and_reset(torch_cuda):
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    spec = ARCHS["stride2_three_groups"]
    _, q8 = _models(spec)
    blob = MF.write_container(q8)
    audio = np.stack([synth_audio(8000, 1300 + i) for i in range(4)])
    dev = torch.from_numpy(audio).cuda()
    a = StreamEngine(blob, n_streams=4)
    first = a.predict_clip(dev[:, :4000].contiguous()).cpu().numpy()
    sd = a.state_dict()
    assert sd["nn"].shape == (4, a.state_elements) and sd["pending"].shape == (4, 1, 40)
    b = StreamEngine(blob, n_streams=4)
    b.load_state_dict(sd)
    assert np.array_equal(a.predict_clip(dev[:, 4000:].contiguous()).cpu().numpy(), b.predict_clip(dev[:, 4000:].contiguous()).cpu().numpy())
    # reset: quantised rings hold the zero point of the tensor they buffer -> same scores as a fresh engine
    a.reset()
    assert np.array_equal(a.predict_clip(dev[:, :4000].contiguous()).cpu().numpy(), first)
    a.reset(stream_ids=[1])
    c = StreamEngine(blob, n_streams=4)
    st_a, st_c = a.state_dict(), c.state_dict()
    assert np.array_equal(st_a["nn"][1], st_c["nn"][1]) and np.array_equal(st_a["carry"][1], st_c["carry"][1])


def test_okay_nabu_through_the_generic_path_equals_the_compiled_in_kernels(torch_cuda):
    """MWW_FORCE_GENERIC=1 sends the okay_nabu container through the run-time-geometry kernels: int8 scores identical to the
    tensor-core path, fp32 within the summation-order tolerance."""
    from microwakeword_b200.engine import StreamEngine
    from conftest import GOLDEN
    torch = torch_cuda
    audio = np.stack([synth_audio(16000, 1400 + i) for i in range(6)])
    dev = torch.from_numpy(audio).cuda()
    for kind in ("f32", "int8"):
        blob = open(os.path.join(GOLDEN, "okay_nabu_synth_%s.mww" % kind), "rb").read()
        fast = StreamEngine(blob, n_streams=6).predict_clip(dev).cpu().numpy()
        os.environ["MWW_FORCE_GENERIC"] = "1"
        try:
            gen = StreamEngine(blob, n_streams=6)
        finally:
            del os.environ["MWW_FORCE_GENERIC"]
        slow = gen.predict_clip(dev).cpu().numpy()
        assert np.array_equal(slow, fast) if kind == "int8" else np.abs(slow - fast).max() <= 1e-5
