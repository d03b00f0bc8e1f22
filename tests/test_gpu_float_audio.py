"""float32 device audio through every frontend variant (run with -m gpu on an H100).

The float entry points (mww_features_f32 / mww_predict_clip_f32, reached through StreamEngine.features / predict_clip with a
float32 tensor) convert each sample inside the frontend kernels.  Their contract: exactly what the int16 entry points give on
audio_utils.to_int16 of the same audio -- bit-identical uint16 features, probabilities and state_dict() -- for the fp32 and the
int8 model, in every kernel variant that reads caller audio, on aligned and unaligned tensors.

Audio: P distinct base streams of random float audio (per-stream amplitudes from -80 dBFS to clipping), salted with the values
the CPU conversion test checks (every float within 2 ulp of an integer boundary, NaNs, infinities, subnormals, +-0, +-FLT_MAX);
stream s carries base[s % P].  Stream counts give each kernel's grid at least three waves with a partial last one."""

import os

import numpy as np
import pytest

from conftest import GOLDEN
from microwakeword_b200.audio.audio_utils import to_int16

pytestmark = pytest.mark.gpu

P = 1021                       # prime: stream s and the stream a CTA handled one wave earlier carry different audio
N_TOTAL = 64000

# Upper bounds on CTAs per SM (so the wave counts below are lower bounds), and streams per CTA at the shapes used here.  The
# K1-family kernels take 50.6 KB of shared memory each, so at most 4 fit an SM; register counts from -Xptxas -v.
OCCUPANCY = {
    "clip_fused": (4, 1),      # k1_spectral_kernel<true, 4>: <= 64 registers
    "k1_clip": (3, 1),         # k1_spectral_kernel<false, 3> (MWW_NO_FUSE): __launch_bounds__(256, 3), 80 registers
    "hop": (3, 1),             # k1_spectral_hop_kernel: 72 registers
    "live_fused": (4, 5),      # k1k2_packed_kernel, 3 frames per call: k1_packed_streams(3) = 5 streams per CTA, 64 registers
    "k1_live": (3, 5),         # k1_spectral_packed_kernel (MWW_NO_FUSE), 3 frames per call: 72 registers
    "carry": (16, 1),          # carry_update_kernel: 128 threads, 2048 threads per SM
}


def stream_count(sms, kernels):
    """Smallest count >= 3 waves of every listed kernel's grid (+37) whose last wave is partial in each of them."""
    S = max(3 * occ * sms * spc for occ, spc in (OCCUPANCY[k] for k in kernels)) + 37

    def partial(S):
        return all(-(-S // OCCUPANCY[k][1]) % (OCCUPANCY[k][0] * sms) != 0 for k in kernels)
    while not partial(S):
        S += 1
    for k in kernels:
        occ, spc = OCCUPANCY[k]
        assert -(-S // spc) >= 3 * occ * sms, (k, S)
    return S


def _salt(rng):
    k = rng.integers(-32770, 32771, 4096)
    centre = (k / 32768.0).astype(np.float32)
    near = [centre]
    for direction in (np.inf, -np.inf):
        x = centre
        for _ in range(2):
            x = np.nextafter(x, np.float32(direction))
            near.append(x)
    special = np.concatenate([np.array([0.0, -0.0, np.inf, -np.inf, np.finfo(np.float32).max, -np.finfo(np.float32).max,
                                        0.99999994, 3.0517578e-05], np.float32),
                              np.array([0x7FC00000, 0xFFC00000, 0x7F800001, 0x7FA5A5A5, 0x00000001, 0x807FFFFF],
                                       np.uint32).view(np.float32)])
    return np.concatenate(near + [np.repeat(special, 64)])


@pytest.fixture(scope="module")
def audio(torch_cuda):
    """(base float32 [P, N_TOTAL] CUDA, its to_int16 [P, N_TOTAL] CUDA).  Chunks are gathered per call (see _chunk)."""
    rng = np.random.default_rng(42)
    amp = (10.0 ** rng.uniform(-4.0, 0.3, P)).astype(np.float32)[:, None]       # -80 dBFS .. 2x full scale (clipping)
    base = (rng.standard_normal((P, N_TOTAL), dtype=np.float32) * amp).astype(np.float32)
    salt = _salt(rng)
    pos = rng.random((P, N_TOTAL)) < 0.02
    base[pos] = salt[rng.integers(0, salt.size, int(pos.sum()))]
    with np.errstate(invalid="ignore", over="ignore"):
        i16 = to_int16(base)
    return torch_cuda.from_numpy(base).cuda(), torch_cuda.from_numpy(i16).cuda()


def _chunk(torch, base, S, pos, n):
    idx = torch.arange(S, device="cuda") % P
    return base[:, pos:pos + n].index_select(0, idx).contiguous()


def _unaligned(torch, x, offset, pitch_extra):
    """x [S, n] -> the same values in a tensor whose storage starts `offset` elements in and whose row pitch is n + pitch_extra."""
    S, n = x.shape
    pitch = n + pitch_extra
    flat = torch.full((S * pitch + offset,), float("nan"), dtype=x.dtype, device=x.device)
    view = flat[offset:].view(S, pitch)[:, :n]
    view.copy_(x)
    assert view.storage_offset() == offset and view.stride() == (pitch, 1)
    return view


def _blob(model):
    with open(os.path.join(GOLDEN, "okay_nabu_synth_%s.mww" % model), "rb") as f:
        return f.read()


def _bits(torch, t):
    """float32 / uint16 CUDA tensor -> its bits as int32 / int16 (NaN-safe, and torch.equal has no uint16 kernel)"""
    return t.contiguous().view({torch.float32: torch.int32, torch.uint16: torch.int16}[t.dtype])


def _same_state(a, b):
    assert a.keys() == b.keys()
    for k in a:
        if isinstance(a[k], np.ndarray):
            assert a[k].dtype == b[k].dtype and np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)), k
        else:
            assert a[k] == b[k], k


def run_and_compare(torch, audio, model, S, schedule, hop=160, layout=None):
    """schedule: list of (n_samples, dtype of the call on the float handle: "f32" or "i16").  A model handle and a frontend-only
    handle take the float calls; twins of both take to_int16 of the same samples as int16.  Every call's probabilities and
    features, and the final state of all four, must be bit-identical."""
    from microwakeword_b200.engine import StreamEngine
    base_f32, base_i16 = audio
    blob = _blob(model)
    eng_f, eng_i = StreamEngine(blob, n_streams=S), StreamEngine(blob, n_streams=S)
    fe_f, fe_i = StreamEngine(None, n_streams=S), StreamEngine(None, n_streams=S)
    if hop != 160:
        for e in (eng_f, eng_i, fe_f, fe_i):
            e.set_window_step(hop)
    pos = 0
    for call, (n, kind) in enumerate(schedule):
        x_i = _chunk(torch, base_i16, S, pos, n)
        x_f = x_i if kind == "i16" else _chunk(torch, base_f32, S, pos, n)
        if kind == "f32" and layout is not None:
            x_f = _unaligned(torch, x_f, *layout)
        p_f, p_i = eng_f.predict_clip(x_f), eng_i.predict_clip(x_i)
        assert p_f.shape == p_i.shape and torch.equal(_bits(torch, p_f), _bits(torch, p_i)), ("probabilities", call, n, kind)
        r_f, r_i = fe_f.features(x_f), fe_i.features(x_i)
        assert r_f.shape == r_i.shape and torch.equal(_bits(torch, r_f), _bits(torch, r_i)), ("features", call, n, kind)
        pos += n
    assert pos <= N_TOTAL
    _same_state(eng_f.state_dict(), eng_i.state_dict())
    _same_state(fe_f.state_dict(), fe_i.state_dict())


LIVE = [(480, "f32")] * 12                                   # 1 frame, then 3 frames per call: the fused short-call kernel
CLIP = [(48000, "f32"), (16000, "f32")]                      # 3 s, then 1 s entering with 320 buffered samples
CLIP_THEN_LIVE = [(16000, "f32")] + [(480, "f32")] * 10
ALTERNATING = [(480, k) for k in ("f32", "i16") * 5] + [(16000, "f32"), (480, "i16"), (16000, "i16")] + \
              [(480, k) for k in ("f32", "i16") * 3]
MODELS = ("f32", "int8")


@pytest.mark.parametrize("model", MODELS)
def test_live_sequence(torch_cuda, audio, model):
    sms = torch_cuda.cuda.get_device_properties(0).multi_processor_count
    run_and_compare(torch_cuda, audio, model, stream_count(sms, ["live_fused"]), LIVE)


@pytest.mark.parametrize("model", MODELS)
def test_clip_calls(torch_cuda, audio, model):
    sms = torch_cuda.cuda.get_device_properties(0).multi_processor_count
    run_and_compare(torch_cuda, audio, model, stream_count(sms, ["clip_fused", "carry"]), CLIP)


@pytest.mark.parametrize("model", MODELS)
def test_unfused_kernels(torch_cuda, audio, model, monkeypatch):
    """MWW_NO_FUSE: K1 (per-stream and packed forms), K2 and the separate carry update, for a clip and live calls."""
    monkeypatch.setenv("MWW_NO_FUSE", "1")                   # read at mww_create
    sms = torch_cuda.cuda.get_device_properties(0).multi_processor_count
    run_and_compare(torch_cuda, audio, model, stream_count(sms, ["k1_clip", "k1_live", "carry"]), CLIP_THEN_LIVE)


@pytest.mark.parametrize("model", MODELS)
def test_hop_320(torch_cuda, audio, model):
    sms = torch_cuda.cuda.get_device_properties(0).multi_processor_count
    run_and_compare(torch_cuda, audio, model, stream_count(sms, ["hop", "carry"]), CLIP_THEN_LIVE, hop=320)


@pytest.mark.parametrize("model", MODELS)
def test_alternating_int16_and_float_calls(torch_cuda, audio, model):
    sms = torch_cuda.cuda.get_device_properties(0).multi_processor_count
    run_and_compare(torch_cuda, audio, model, stream_count(sms, ["live_fused", "clip_fused", "carry"]), ALTERNATING)


@pytest.mark.parametrize("offset,pitch_extra", [(1, 3), (2, 1), (3, 2), (0, 5)])
@pytest.mark.parametrize("model", MODELS)
def test_unaligned_float_tensors(torch_cuda, audio, model, offset, pitch_extra):
    """Storage offsets of 1 to 3 floats and row pitches that are not a multiple of 4 take the per-sample loaders."""
    sms = torch_cuda.cuda.get_device_properties(0).multi_processor_count
    schedule = [(480, "f32")] * 4 + [(16000, "f32")] + [(480, "f32")] * 3
    run_and_compare(torch_cuda, audio, model, stream_count(sms, ["live_fused", "clip_fused", "carry"]), schedule,
                    layout=(offset, pitch_extra))


def test_other_dtypes_and_host_tensors_are_refused(torch_cuda):
    from microwakeword_b200.engine import StreamEngine
    from microwakeword_b200.inference import Model
    torch = torch_cuda
    eng = StreamEngine(_blob("f32"), n_streams=4)
    bad = [torch.zeros((4, 480), dtype=dt, device="cuda") for dt in (torch.float64, torch.float16, torch.bfloat16, torch.int32)]
    bad.append(torch.zeros((4, 480), dtype=torch.float32))                    # host tensor
    for x in bad:
        for fn in (eng.features, eng.predict_clip, eng.step):
            with pytest.raises(ValueError):
                fn(x)
    assert eng.frontend_buffered == 0 and eng.pending_rows == 0
    # Model.step takes the device form too: float32 CUDA audio gives what its int16 conversion gives
    m_f, m_i = Model(os.path.join(GOLDEN, "okay_nabu_synth_int8.mww"), batch=3), Model(os.path.join(GOLDEN, "okay_nabu_synth_int8.mww"), batch=3)
    x = torch.rand((3, 4800), device="cuda") * 2.2 - 1.1
    with np.errstate(invalid="ignore", over="ignore"):
        x_i = torch.from_numpy(to_int16(x.cpu().numpy())).cuda()
    assert torch.equal(m_f.step(x), m_i.step(x_i))
