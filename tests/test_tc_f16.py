"""The wgmma clip kernel's fp16 first conv: integer features times fp16 hi / lo weights (mww_nn_tc.cu, mww_nn_tc_prep.h).

CPU: the fp16 K-slot layout reads back to the scaled weights to within fp16 hi / lo precision and is the hardware's 128-byte
swizzle; the largest feature the frontend can emit, derived from its log table, is exact in fp16; the first conv's weight scale
admits the shipped model and refuses one whose output channels span more than the scheme keeps.
GPU: at the benchmark's shape the fp16 kernel is no further from the fp32 oracle than the 3xTF32 kernel (MWW_TC_TF32=1), and
leaves the same ring state to within 1e-5; it holds across chunk boundaries and pending rows; and a model whose weights
refuse fp16, a handle fed rows by infer_features and one whose state was set from outside all run the 3xTF32 kernel bit for bit."""

import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, ROOT

CSRC = os.path.join(ROOT, "microwakeword_b200", "csrc")
SHIM = r"""
#include "mww_nn_tc_prep.h"
using namespace mww;
extern "C" {
unsigned shim_sw128_off_h(int row, int kk) { return sw128_off_h(row, kk); }
long long shim_layout_f16(const float *w, int K, int N, double mul, int s, unsigned char *out, long long cap) {
    std::vector<unsigned char> blob;
    tc_layout_f16(w, K, N, mul, s, &blob);
    if (out && (long long)blob.size() <= cap) memcpy(out, blob.data(), blob.size());
    return (long long)blob.size();
}
int shim_scale_exp(double m) { return f16_scale_exp(m); }
int shim_max_feature() { return kTcMaxFeature; }
int shim_fresh_steps() { return kTcFreshSteps; }
int shim_scales(const float *w0, int *s_fc) {
    const TcF16Scales r = tc_f16_scales(w0);
    *s_fc = r.s_fc;
    return r.ok;
}
}
"""


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    d = tmp_path_factory.mktemp("tc_f16")
    src, so = str(d / "shim.cc"), str(d / "shim.so")
    with open(src, "w") as f:
        f.write(SHIM)
    res = subprocess.run(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-I", CSRC, "-o", so, src], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    L = ctypes.CDLL(so)
    L.shim_sw128_off_h.restype = ctypes.c_uint
    L.shim_layout_f16.restype = ctypes.c_longlong
    L.shim_layout_f16.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_double, ctypes.c_int, ctypes.c_void_p, ctypes.c_longlong]
    L.shim_scale_exp.argtypes = [ctypes.c_double]
    return L


def _model(name):
    with open(os.path.join(GOLDEN, name), "rb") as f:
        return f.read()


def _scales(L, w0):
    """tc_f16_scales of first-conv weights [200, 32]: (ok, s_fc)."""
    w0 = np.ascontiguousarray(w0, np.float32).reshape(200, 32)
    s = ctypes.c_int(0)
    ok = L.shim_scales(w0.ctypes.data_as(ctypes.c_void_p), ctypes.byref(s))
    return bool(ok), s.value


def test_fp16_operand_layout_round_trips_and_is_a_swizzle_bijection(shim):
    """64 fp16 per 128-byte row, the eight 16-byte chunks of a row permuted by (row & 7); the planes read back through the same
    map give hi + lo within 2^-22 |x| (+ the subnormal floor 2^-25) of x = w * mul * 2^s, hi and lo are fp16 values, |hi| <= 2^15,
    and the tail of the last slot is zero."""
    L = shim
    for rows in (32, 64, 128):
        off = np.array([[L.shim_sw128_off_h(r, kk) for kk in range(64)] for r in range(rows)], np.int64)
        assert np.array_equal(np.sort(off.ravel()), 2 * np.arange(rows * 64))
        assert all(np.array_equal(np.sort(off[r]), r * 128 + 2 * np.arange(64)) for r in range(rows))
        assert np.array_equal((off % 128) // 16, (np.arange(64)[None, :] // 8) ^ (np.arange(rows)[:, None] & 7))
    rng = np.random.default_rng(3)
    for K, N, mul in ((200, 32, 0.0390625), (32, 64, 1.0), (64, 64, 1.0)):
        w = (rng.standard_normal((K, N)) * rng.choice([1e-3, 1.0, 50.0], (K, N))).astype(np.float32)
        x64 = w.astype(np.float64) * mul
        s = L.shim_scale_exp(float(np.abs(x64).max()))
        x = x64 * 2.0 ** s
        assert 2.0 ** 14 <= np.abs(x).max() < 2.0 ** 15
        n = L.shim_layout_f16(w.ctypes.data_as(ctypes.c_void_p), K, N, mul, s, None, 0)
        slots, plane = (K + 63) // 64, N * 128
        assert n == slots * 2 * plane
        blob = np.zeros(n, np.uint8)
        L.shim_layout_f16(w.ctypes.data_as(ctypes.c_void_p), K, N, mul, s, blob.ctypes.data_as(ctypes.c_void_p), n)
        h = blob.view(np.float16)
        hi, lo = np.zeros((slots * 64, N), np.float64), np.zeros((slots * 64, N), np.float64)
        for k in range(slots * 64):
            for col in range(N):
                o = (k // 64) * 2 * plane + L.shim_sw128_off_h(col, k % 64)
                hi[k, col], lo[k, col] = h[o // 2], h[(o + plane) // 2]
        assert not hi[K:].any() and not lo[K:].any()
        assert np.array_equal(hi[:K], x.astype(np.float16).astype(np.float64))            # hi = fp16(x), round to nearest
        assert (np.abs(hi) <= 2.0 ** 15).all()
        assert (np.abs(hi[:K] + lo[:K] - x) <= np.abs(x) * 2.0 ** -22 + 2.0 ** -25).all()


def _log_lut():
    # mww_tables.cc: the log2 correction table of the frontend's log scale
    x = np.arange(129) / 128.0
    return np.floor(65536.0 * (np.log2(1.0 + x) - x) + 0.5).astype(np.int64)


def test_largest_frontend_feature_is_exact_in_fp16(shim):
    """log_scale (mww_frontend_dev.cuh) of a 32-bit input: log2 = (integer << 16) + frac + c0 + rel with integer <= 31.  Every
    16-bit frac is reachable at integer 31 (x >= 2^31), and any smaller integer part gives a smaller log2 than frac = 0 at 31 plus
    the largest correction, so the maximum over all inputs is the maximum over frac at integer 31 -- 1 420, below 2048."""
    lut = _log_lut()
    frac = np.arange(65536, dtype=np.int64)
    seg = frac >> 9
    c0, c1 = lut[seg], lut[seg + 1]
    rel = ((c1 - c0) * (frac - (seg << 9))) >> 16
    frac_part = frac + c0 + rel

    def feature(integer):
        log2v = (integer << 16) + frac_part
        loge = (45426 * log2v + 32768) >> 16
        return ((loge << 6) + 32768) >> 16

    top = int(feature(31).max())
    assert int(feature(30).max()) <= int(feature(31).min()) <= top
    assert top == shim.shim_max_feature() == 1420 and top <= 2048


def test_fresh_steps_replace_the_first_conv_ring_and_pending_rows(shim):
    """After a call of kTcFreshSteps steps the first-conv ring (the 2 rows before the first unconsumed one) and the pending rows
    are the call's own rows, whatever 0..2 rows were pending when it started."""
    k = shim.shim_fresh_steps()
    for pend in range(3):
        for rows in range(3 * k - pend, 3 * k - pend + 3):           # exactly k steps
            assert (pend + rows) // 3 == k and 3 * k - 2 >= pend
    assert k == 2


def test_scales_admit_the_shipped_model_and_refuse_a_channel_out_of_range(shim):
    from microwakeword_b200 import model_file
    w0 = np.asarray(model_file.read_container(_model("okay_nabu_synth_f32.mww"))["first_conv/w"], np.float32).reshape(200, 32)
    ok, s = _scales(shim, w0)
    assert ok and 2.0 ** 14 <= np.abs(w0.astype(np.float64) * 0.0390625).max() * 2.0 ** s < 2.0 ** 15
    assert not _scales(shim, _scaled_channel(w0))[0]
    bad = w0.copy()
    bad[3, 3] = np.nan
    assert not _scales(shim, bad)[0]


# ---- GPU -------------------------------------------------------------------------------------------------------------------

def _engine(blob, S, tf32, monkeypatch):
    from microwakeword_b200.engine import StreamEngine
    if tf32:
        monkeypatch.setenv("MWW_TC_TF32", "1")        # read at mww_create
    else:
        monkeypatch.delenv("MWW_TC_TF32", raising=False)
    eng = StreamEngine(blob, n_streams=S)
    monkeypatch.delenv("MWW_TC_TF32", raising=False)
    return eng


@pytest.mark.gpu
def test_fp16_kernel_is_no_further_from_the_oracle_at_benchmark_shape(torch_cuda, monkeypatch):
    """bench.py's step (65 536 streams, two 3 s predict_clip calls) on the fp16 and on the 3xTF32 kernel: the largest |dp| against
    the fp32 oracle (fp16 not worse beyond 2^-24 of rounding noise, both within 1e-5) and the largest difference of the ring state
    the two leave (relative to max(1, |v|)).  The two kernels must really differ: the probabilities are not bit-identical."""
    import oracle
    from test_gpu_full_size import P_AUDIO, _base_audio, periodic_streams
    torch = torch_cuda
    S, N = 65536, 48000
    blob = _model("okay_nabu_synth_f32.mww")
    base = _base_audio(P_AUDIO, N, 7000)
    dev = periodic_streams(torch, base, S, ("clip_tc",))
    _, want = oracle.run_pipeline(blob, np.concatenate([base, base], 1), want_features=False, threads=8)
    idx = torch.arange(S, device="cuda") % P_AUDIO
    w = torch.from_numpy(np.ascontiguousarray(want[:, :199], np.float32)).cuda().index_select(0, idx)
    res = {}
    for tf32 in (False, True):
        eng = _engine(blob, S, tf32, monkeypatch)
        p = torch.cat([eng.predict_clip(dev).clone() for _ in range(2)], 1)
        res[tf32] = (p, (p - w).abs().max().item(), eng.state_dict()["nn"].astype(np.float64))
        del eng
    ring = res[True][2]
    ring_diff = float((np.abs(res[False][2] - ring) / np.maximum(np.abs(ring), 1.0)).max())
    print("largest |dp| vs the fp32 oracle: fp16 %.3g, 3xTF32 %.3g; ring state fp16 vs 3xTF32 %.3g" % (res[False][1], res[True][1], ring_diff))
    assert res[False][1] <= 1e-5 and res[True][1] <= 1e-5
    assert res[False][1] <= res[True][1] + 2.0 ** -24
    assert ring_diff <= 1e-5
    assert not torch.equal(res[False][0], res[True][0])


# predict calls (samples after the first call's 480-sample window): rows per call, entering with 0, 1 and 2 pending rows and ending on
# both sides of the 128-step chunks; the 8-step call runs the mma.sync kernel
PREDICT_ROWS = [48, 193, 196, 379, 384, 26, 385, 772]


@pytest.mark.gpu
def test_fp16_kernel_across_chunks_and_pending_rows(torch_cuda):
    """predict_clip through calls of 16 .. 257 steps on 2 x SMs + 37 streams (some CTAs take a second stream): within 1e-5 of the
    oracle over the same audio, streams with the same content bit-identical."""
    import oracle
    from microwakeword_b200.engine import StreamEngine
    from test_gpu_full_size import P_ROWS, _base_audio, check_streams, periodic_streams
    torch = torch_cuda
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    S = 2 * sms + 37
    total = sum(PREDICT_ROWS)
    blob = _model("okay_nabu_synth_f32.mww")
    audio = _base_audio(P_ROWS, 480 + 160 * (total - 1), 8100)
    _, want = oracle.run_pipeline(blob, audio, want_features=False, threads=8)
    dev = torch.from_numpy(audio).cuda().index_select(0, torch.arange(S, device="cuda") % P_ROWS)
    eng = StreamEngine(blob, n_streams=S)
    got, pos = [], 0
    for i, r in enumerate(PREDICT_ROWS):
        n = 480 + 160 * (r - 1) if i == 0 else 160 * r
        got.append(eng.predict_clip(dev[:, pos:pos + n].contiguous()))
        pos += n
    assert [g.shape[1] for g in got] == [16, 64, 65, 127, 128, 8, 129, 257]
    check_streams(torch, torch.cat(got, 1), want, False, "predict sequence")


def _scaled_channel(w0):
    """one first-conv output channel 2^20 below the others: its lo parts would be fp16 subnormals"""
    w0 = np.array(w0, np.float32).reshape(200, 32)
    w0[:, 5] *= np.float32(2.0 ** -20)
    return w0


def _scaled_channel_model():
    from microwakeword_b200 import model_file
    t = dict(model_file.read_container(_model("okay_nabu_synth_f32.mww")))
    t["first_conv/w"] = _scaled_channel(t["first_conv/w"]).reshape(np.asarray(t["first_conv/w"]).shape)
    return model_file.write_container(t)


@pytest.mark.gpu
def test_models_and_handles_outside_the_fp16_bounds_run_3xtf32_bit_for_bit(torch_cuda, monkeypatch):
    """A model whose weights refuse fp16 gives exactly what MWW_TC_TF32=1 gives.  So does a handle for the first predict call after
    an infer_features call, or after a state whose first-conv ring is not made of features was set; a snapshot the library took
    itself keeps the fp16 kernel and continues bit for bit."""
    torch = torch_cuda
    from conftest import synth_audio
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    S = 2 * sms + 1
    audio = torch.from_numpy(np.stack([synth_audio(48000, 9000 + i) for i in range(S)])).cuda()
    clip, short = audio[:, :48000].contiguous(), audio[:, :16000].contiguous()   # 100 steps; then 1 s: 33 steps
    bad = _scaled_channel_model()
    a, b = _engine(bad, S, False, monkeypatch), _engine(bad, S, True, monkeypatch)
    assert torch.equal(a.predict_clip(clip), b.predict_clip(clip))
    del a, b
    blob = _model("okay_nabu_synth_f32.mww")
    orig, b = _engine(blob, S, False, monkeypatch), _engine(blob, S, True, monkeypatch)
    assert not torch.equal(orig.predict_clip(clip), b.predict_clip(clip))   # orig runs the fp16 kernel
    snap = orig.state_dict()
    for how in ("infer", "state"):
        a, b = _engine(blob, S, False, monkeypatch), _engine(blob, S, True, monkeypatch)
        for e in (a, b):
            if how == "infer":
                e.infer(e.features(clip))
            else:
                bent = dict(snap, nn=snap["nn"].copy())
                bent["nn"][:, 7] += np.float32(0.01)          # a first-conv ring entry no feature gives
                e.load_state_dict(bent)
        assert torch.equal(a.predict_clip(short), b.predict_clip(short)), how
        assert np.array_equal(a.state_dict()["nn"], b.state_dict()["nn"]), how
    # the snapshot itself: fp16 again, bit for bit the engine it came from, and not what 3xTF32 gives from it
    c, t = _engine(blob, S, False, monkeypatch), _engine(blob, S, True, monkeypatch)
    c.load_state_dict(snap)
    t.load_state_dict(snap)
    pc = c.predict_clip(short)
    assert torch.equal(orig.predict_clip(short), pc) and not torch.equal(pc, t.predict_clip(short))
