"""Hybrid models on the CPU: the float streaming .tflite the reference writes with quantize=False (utils.py:328: dynamic-range
quantisation, large CONV_2D / DEPTHWISE_CONV_2D / FULLY_CONNECTED weights stored as per-channel int8 and run by TFLite's
hybrid kernels).
  * known answers of the two input quantisers, oracle and device formulation;
  * the loader: round trips in each writer mode, refusals, the float graph that no longer reads int8 codes as floats;
  * the generic hybrid kernel's phase functions executed thread by thread (tests/host_emul/emul_hybrid.cc) are bit-identical
    to the hybrid oracle (tests/hybrid_ref), probabilities and rings, over ragged call sequences on several geometries;
  * the batched-evaluation warm-up rule holds on a hybrid model;
  * the hybrid kernel compiles for sm_90a without spills or a stack frame.
The GPU side is tests/test_zz_hybrid_gpu.py."""

import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import oracle
import hybrid_ref as HR
import tflite_hybrid_writer as HW
import tflite_writer as TW
from conftest import GOLDEN, synth_audio
from host_emul import emul_hybrid as EH
from microwakeword_b200 import batched
from microwakeword_b200 import model_file as MF
from microwakeword_b200 import tflite_file as TF
from oracle import mixednet_ref as R


def converter_rule(op, n):
    return n >= 1024                                   # the converter's dynamic-range threshold (elements)


def all_rule(op, n):
    return True


GEOMS = {
    # okay_nabu, converter threshold: first conv, the four 1x1 convs, block 4's depthwise conv and the head are hybrid
    "okay_nabu": (R.Spec(), converter_rule, True),
    # every op hybrid, three MixConv groups, dense head with symmetric input quantisation
    "stride2_three_groups": (R.Spec(16, 6, 2, (40,), ((7, 11, 13),), head_rows=9), all_rule, False),
    # MixConv [9, 33] on 64 channels: 288 and 1056 elements fall on opposite sides of the threshold; float head
    "split_threshold": (R.Spec(64, 5, 3, (32, 48), ((9, 33), (3,)), head_rows=5), converter_rule, True),
}


def hybrid_tensors(spec, rule, fc_asym=True, seed=0):
    f32 = R.fold_bn(spec, R.init_synthetic(spec, seed))
    return TF.tensors_from_tflite(HW.write_hybrid_mixednet(f32, rule, fc_asym))


def _features(n_streams, n_samples, seed):
    audio = np.stack([synth_audio(n_samples, seed + i) for i in range(n_streams)])
    feats, _ = oracle.run_pipeline(None, audio, want_probs=False)
    return feats


# ------------------------------------------------------------------------------------------------------ quantiser KATs
# hand-worked: rmin = min(0, min x), rmax = max(0, max x), scale = (rmax - rmin) / 255, zero point from the side with the
# smaller error term, q = round_half_away((float)zp + x * (1 / scale)); symmetric: q = round(x * (127 / range))
ASYM_KATS = [
    # all zeros: codes 0, scale 1, zero point 0
    ([0.0, 0.0, 0.0], [0, 0, 0], 1.0, 0),
    # all positive: rmin 0, scale 1, zero point -128 (from the min side); -125.5 rounds away from zero to -126
    ([1.0, 2.5, 255.0], [-127, -126, 127], 1.0, -128),
    # all negative: rmax 0, scale 1, zero point 127 (from the max side); 124.5 rounds to 125
    ([-255.0, -1.0, -2.5], [-128, 126, 125], 1.0, 127),
    # nudged zero point, min branch: rmin -1, rmax 3 -> -128 + 63.75 = -64.25 -> -64
    ([-1.0, 3.0, 0.5], [-128, 127, -32], np.float32(4.0 / 255.0), -64),
    # nudged zero point, max branch: rmin -3, rmax 1 -> 127 - 63.75 = 63.25 -> 63
    ([-3.0, 1.0, -0.5], [-128, 127, 31], np.float32(4.0 / 255.0), 63),
    # exact .5 ties at scale 1, zero point -128: -127.5 -> -128, -126.5 -> -127, -125.5 -> -126, 126.5 -> 127
    ([0.5, 1.5, 2.5, 254.5, 255.0], [-128, -127, -126, 127, 127], 1.0, -128),
    # a single non-zero value
    ([0.0, 0.0, 0.75, 0.0], [-128, -128, 127, -128], np.float32(0.75 / 255.0), -128),
    ([0.0, -2.0, 0.0], [127, -128, 127], np.float32(2.0 / 255.0), 127),
]
SYM_KATS = [
    ([0.0, 0.0], [0, 0], 1.0),
    # range 127 -> 1 / scale = 1; ties 0.5 -> 1, -1.5 -> -2, 2.5 -> 3 (half away from zero)
    ([127.0, 0.5, -1.5, 2.5], [127, 1, -2, 3], 1.0),
    ([-2.0, 1.0, 0.5, 2.0], [-127, 64, 32, 127], np.float32(2.0) / np.float32(127.0)),
    ([0.0, -3.0], [0, -127], np.float32(3.0) / np.float32(127.0)),
]


@pytest.mark.parametrize("impl", ["oracle", "device_phases"])
def test_asymmetric_quantiser_known_answers(impl):
    fn = HR.quantize if impl == "oracle" else EH.quantize
    for x, q, scale, zp in ASYM_KATS:
        got_q, got_s, got_zp = fn(np.asarray(x, np.float32))
        assert list(got_q) == q and got_s == np.float32(scale) and got_zp == zp, (x, got_q, got_s, got_zp)


@pytest.mark.parametrize("impl", ["oracle", "device_phases"])
def test_symmetric_quantiser_known_answers(impl):
    fn = HR.quantize if impl == "oracle" else EH.quantize
    for x, q, scale in SYM_KATS:
        got_q, got_s, got_zp = fn(np.asarray(x, np.float32), symmetric=True)
        assert list(got_q) == q and got_s == np.float32(scale) and got_zp == 0, (x, got_q, got_s)


def test_device_quantiser_equals_the_oracle_on_random_tensors():
    rng = np.random.default_rng(5)
    for i in range(300):
        n = int(rng.integers(1, 3000))
        x = (rng.standard_normal(n) * 10.0 ** rng.uniform(-4, 3)).astype(np.float32)
        if i % 3 == 0:
            x = np.maximum(x, 0)                                         # post-ReLU tensors
        for sym in (False, True):
            a, b = HR.quantize(x, sym), EH.quantize(x, sym)
            assert np.array_equal(a[0], b[0]) and a[1] == b[1] and a[2] == b[2]


# ------------------------------------------------------------------------------------------------------------- loader
@pytest.mark.parametrize("name", list(GEOMS))
def test_loader_reads_hybrid_ops_per_op(name):
    spec, rule, fc_asym = GEOMS[name]
    f32 = R.fold_bn(spec, R.init_synthetic(spec, 0))
    got = TF.tensors_from_tflite(HW.write_hybrid_mixednet(f32, rule, fc_asym))
    arch = MF.Arch.decode(got["arch"])
    slots = MF.hybrid_slots(arch)
    assert MF.is_hybrid(got) and not MF.is_quantized(got) and np.array_equal(got["arch"], spec.encode())
    sizes = {"first_conv": f32["first_conv/w"].size, "head": f32["head/w"].size}
    for b in range(arch.n_blocks):
        sizes["b%d/pw" % b] = f32["b%d/pw/w" % b].size
    want = []
    for s in slots:
        if s.startswith("b") and "/dw" in s:
            b, j = int(s[1:s.index("/")]), int(s[s.index("/dw") + 3:])
            cin = arch.block_in_channels(b)
            g = len(arch.mixconv_kernel_sizes[b])
            n = cin // g + (cin % g if j == 0 else 0)
            n *= arch.mixconv_kernel_sizes[b][j]
        else:
            n = sizes[s]
        hy = rule(s, n)
        want.append(0 if not hy else (MF.HYBRID_SYMMETRIC if s == "head" and not fc_asym else MF.HYBRID_ASYMMETRIC))
    assert list(got["hy/mode"]) == want
    # fp32 tensors hold the dequantised weights; each is within half a step of the original
    for key, hyk in (("first_conv/w", "hy/first_conv"), ("head/w", "hy/head")):
        if hyk + "/w" in got:
            s = got[hyk + "/scale"]
            assert np.array_equal(got[key], (got[hyk + "/w"].astype(np.float32) * s).astype(np.float32))
            assert np.abs(got[key] - f32[key]).max() <= s.max() / 2 * 1.0001
    if name == "split_threshold":
        assert list(got["hy/mode"][1:3]) == [0, 1]                       # 288 elements float, 1056 hybrid
        assert np.all(got["hy/b0/dw/w"][:, :32] == 0) and np.all(got["hy/b0/dw/scale"][:32] == 0)
        assert np.array_equal(got["b0/dw/w"][:, :32], f32["b0/dw/w"][:, :32])


def test_pure_float_graph_gives_todays_container():
    f32 = MF.load(os.path.join(GOLDEN, "okay_nabu_synth_f32.mww"))
    plain = TW.write_streaming_mixednet(f32)
    got = TF.tensors_from_tflite(plain)
    assert not MF.is_hybrid(got) and not any(k.startswith("hy/") for k in got)
    assert MF.write_container(got) == MF.write_container(TF.tensors_from_tflite(plain))
    for k, v in f32.items():
        if k in got:
            assert np.array_equal(got[k], v), k


def test_float_graph_never_reads_int8_codes_as_floats():
    """okay_nabu_synth_f32.mww in a float graph whose >= 1024-element kernels are per-channel int8: a hybrid container whose
    fp32 tensors are the dequantised weights, not integer-valued floats."""
    f32 = MF.load(os.path.join(GOLDEN, "okay_nabu_synth_f32.mww"))
    got = TF.tensors_from_tflite(HW.write_hybrid_mixednet(f32, converter_rule))
    assert MF.is_hybrid(got)
    assert list(got["hy/mode"]) == [1, 0, 1, 0, 0, 1, 0, 0, 1, 1, 1, 1]
    for k in ("first_conv/w", "head/w", "b3/dw/w", "b0/pw/w"):
        assert np.abs(got[k]).max() < 1.0 and np.abs(got[k] - f32[k]).max() < 0.01, k
    HR.HybridNet(MF.write_container(got))                           # a well-formed hybrid container
    assert not oracle.MixedNet(MF.write_container(got)).is_quantized


def _graph_with(mutate, f32=None, rule=all_rule):
    """a hybrid okay_nabu graph whose tensors `mutate(tensor_dict_by_name)` edits before serialisation"""
    f32 = f32 if f32 is not None else MF.load(os.path.join(GOLDEN, "okay_nabu_synth_f32.mww"))
    return HW.write_hybrid_mixednet(f32, rule, edit=mutate)


def _per_tensor(t, gw):
    t["scale"] = np.asarray([np.max(t["scale"])], np.float32)
    t["zero_point"] = np.zeros(1, np.int64)


def _nonzero_zp(t, gw):
    t["zero_point"] = np.ones(np.size(t["zero_point"]), np.int64)


def _wrong_dim(t, gw):
    t["qdim"] = 0 if t["qdim"] == 3 else 3


def _int16_weights(t, gw):
    raw = np.frombuffer(gw.buffers[t["buffer"]], np.int8).astype(np.int16)
    gw.buffers[t["buffer"]] = raw.tobytes()
    t["type"] = 7


def _int32_bias(t, gw):
    raw = np.frombuffer(gw.buffers[t["buffer"]], np.float32).astype(np.int32)
    gw.buffers[t["buffer"]] = raw.tobytes()
    t["type"] = TW.T_INT32


@pytest.mark.parametrize("tensor,edit,op", [
    ("stream/conv2d/kernel", _per_tensor, "CONV_2D"),
    ("dw_3_0/kernel", _per_tensor, "DEPTHWISE_CONV_2D"),
    ("pw_1/kernel", _nonzero_zp, "CONV_2D"),
    ("pw_2/kernel", _wrong_dim, "CONV_2D"),
    ("dw_1_1/kernel", _wrong_dim, "DEPTHWISE_CONV_2D"),
    ("dense/kernel", _int16_weights, "FULLY_CONNECTED"),
    ("pw_0/bias", _int32_bias, "CONV_2D"),
])
def test_unsupported_weight_forms_are_refused_naming_the_operator(tensor, edit, op):
    blob = _graph_with(lambda ts, gw: edit(ts[tensor], gw))
    with pytest.raises(TF.TfliteError, match=r"\(%s\)" % op):
        TF.tensors_from_tflite(blob)


def test_dequantize_fed_weights_stay_refused():
    """float16 / DEQUANTIZE-fed weights: DEQUANTIZE is outside the streaming op set"""
    f32 = MF.load(os.path.join(GOLDEN, "okay_nabu_synth_f32.mww"))
    TW.OPS["DEQUANTIZE"] = 6
    try:
        def add_dq(ts, gw):
            src = ts["dense/kernel"]
            idx = gw.tensors.index(src)
            w = gw.tensor("dense/kernel_f32", src["shape"], np.float32)
            gw.ops.insert(1, ("DEQUANTIZE", [idx], [w], {}))
            for n, (name, ins, outs, o) in enumerate(gw.ops):
                if name == "FULLY_CONNECTED":
                    gw.ops[n] = (name, [w if i == idx else i for i in ins], outs, o)
        blob = _graph_with(add_dq, f32)
    finally:
        del TW.OPS["DEQUANTIZE"]
    with pytest.raises(TF.TfliteError, match="DEQUANTIZE|builtin#6"):
        TF.tensors_from_tflite(blob)


def test_hybrid_container_round_trips_and_reads_as_float():
    t = hybrid_tensors(*GEOMS["split_threshold"][:2])
    back = MF.read_container(MF.write_container(t))
    assert set(back) == set(t) and all(np.array_equal(back[k], t[k]) for k in t)
    assert MF.is_hybrid(back) and not MF.is_quantized(back)


# -------------------------------------------------------------------------------------- device phases against the oracle
@pytest.fixture(params=["ascending", "descending"])
def thread_order(request):
    EH.lib().emul_hy_thread_order(int(request.param == "descending"))
    yield
    EH.lib().emul_hy_thread_order(0)


@pytest.mark.parametrize("name", list(GEOMS))
def test_hybrid_phases_are_bit_identical_to_the_oracle(name, thread_order):
    spec, rule, fc_asym = GEOMS[name]
    t = hybrid_tensors(spec, rule, fc_asym)
    blob = MF.write_container(t)
    s = spec.stride
    feats = _features(2, 8000, 600)                                   # 50 rows per stream
    n_total = feats.shape[1]
    g = EH.GenHybrid(t, 2)
    refs = [HR.HybridNet(blob) for _ in range(2)]
    pend = [np.zeros((0, 40), np.float32) for _ in range(2)]
    cuts = [0, 1, 2, 9, 9 + s - 1, 30, 31, n_total]
    n_probs = 0
    for i, (a, b) in enumerate(zip(cuts[:-1], cuts[1:])):
        rows = feats[:, a:b]
        xf = rows.astype(np.float32) * np.float32(R.FEATURE_SCALE)
        got = g.infer(xf if i % 2 else rows)
        for k in range(2):
            buf = np.concatenate([pend[k], xf[k]])
            want = [refs[k].step(buf[j:j + s])[0] for j in range(0, buf.shape[0] // s * s, s)]
            pend[k] = buf[buf.shape[0] // s * s:]
            assert np.array_equal(got[k], np.asarray(want, np.float32)), (name, i, k)
            assert np.array_equal(g.state[k], refs[k].state()), (name, i, k)
            assert np.array_equal(g.pend[k, :pend[k].size], pend[k].ravel())
        n_probs += got.shape[1]
    assert n_probs == n_total // s
    assert g.sm_bytes <= 200 * 1024


def test_hybrid_differs_from_the_float_model_it_came_from():
    """the hybrid arithmetic is not the fp32 one: same weights, different (but close) probabilities"""
    spec, rule, _ = GEOMS["okay_nabu"]
    t = hybrid_tensors(spec, rule)
    plain = {k: v for k, v in t.items() if not k.startswith("hy/")}
    feats = _features(1, 16000, 900)[0]
    ph = HR.HybridNet(MF.write_container(t)).predict_u16(feats)
    pf = oracle.MixedNet(MF.write_container(plain)).predict_u16(feats)
    assert not np.array_equal(ph, pf) and np.abs(ph - pf).max() < 0.1


# ------------------------------------------------------------------------------------------------------ batched warm-up
def test_warmup_bound_holds_for_a_hybrid_model():
    """W = stride * warmup_steps(arch) rows of warm-up reproduce the sequential hybrid output bit for bit; W - stride do not
    (for at least one of the seeds)."""
    spec, rule, _ = GEOMS["split_threshold"]
    blob = MF.write_container(hybrid_tensors(spec, rule))
    arch = MF.Arch.decode(spec.encode())
    w = batched.warmup_steps(arch)
    run = lambda rows: HR.HybridNet(blob).predict_u16(rows)             # noqa: E731
    tight = False
    for seed in (1, 2, 3):
        rng = np.random.default_rng(seed)
        steps = rng.integers(1, 3 * w, 12)
        p = batched.plan(steps, spec.stride, spec.stride * w, max_streams=3)
        audio = synth_audio(160 * (p.total_steps * spec.stride + 2), 100 * seed)[None, :]
        feats, _ = oracle.run_pipeline(None, audio, want_probs=False)
        rows = feats[0, :p.total_steps * spec.stride]
        seq = run(rows)

        def segmented(warm):
            out = []
            for i in range(p.n_streams):
                a, b = i * p.seg_steps, min((i + 1) * p.seg_steps, p.total_steps)
                ws = 0 if i == 0 else warm
                out.append(run(rows[(a - ws) * spec.stride:b * spec.stride])[ws:])
            return np.concatenate(out)

        assert np.array_equal(segmented(w), seq)
        tight |= not np.array_equal(segmented(w - 1), seq)
    assert tight


# ---------------------------------------------------------------------------------------------------------- compile
def test_hybrid_kernel_compiles_without_spills_or_stack():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc) and shutil.which("nvcc") is None:
        pytest.skip("nvcc not installed")
    nvcc = nvcc if os.path.exists(nvcc) else shutil.which("nvcc")
    src = os.path.join(os.path.dirname(EH.CSRC), "csrc", "mww_nn_generic.cu")
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-cubin", "-Xptxas", "-v",
                            "-o", os.path.join(d, "g.cubin"), src], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    m = re.search(r"Function properties for \S*nn_generic_hybrid_kernel\S*\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads", r.stderr)
    assert m is not None, r.stderr
    assert m.groups() == ("0", "0", "0"), m.group(0)
