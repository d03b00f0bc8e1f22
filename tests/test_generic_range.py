"""The run-time-geometry MixedNet (microwakeword_b200/csrc/mww_nn_generic.cuh) across the range mww_create accepts -- 512
channels (four passes of every 128-thread channel loop), 8 blocks, 64-tap rings, strides up to 64, a stateless model,
shared memory at the 200 KiB cap -- on the CPU: the phase functions executed thread by thread (tests/host_emul) against

  * the C oracle (oracle/mixednet.c): int8 bit for bit, fp32 within 1e-5;
  * a float64 evaluation of the same graph (mixednet_ref.StreamingF64): every ring entry within RING_RTOL * max(1, |v|)
    of the float64 value, and every probability and ring entry inside its running error bound -- a worst case that holds
    for any summation order and is tight only near the input (BOUND_RELIED pins where it is relied on);
  * the NumPy oracle's ring buffers and pending rows.

The oracles themselves are checked against each other here at the same geometries (C == NumPy), and refuse what their
fixed-size buffers cannot hold.  The GPU side is tests/test_zz_generic_range_gpu.py."""

import numpy as np
import pytest

import hybrid_ref as HR
import oracle
from generic_range import (GEOMETRIES, RING_RTOL, SMEM_CAP, all_geometries, bound_tightness, bound_violations, boundary_specs,
                           call_cuts, f64_run, features, models, ring_tolerance_violations)
from host_emul import emul
from microwakeword_b200 import model_file as MF
from oracle import mixednet_ref as R

NAMES = list(GEOMETRIES) + ["boundary"]

# The float64 bound is a worst case: every layer multiplies the error it inherits by sum |w|, so it is only a useful check
# near the input.  These are the rings (and, for the stateless model, the probability) where it is relied on, with the
# ceiling its median bound / |value| must stay under after 3 s of audio; everywhere else the rings are held to RING_RTOL of
# the float64 values instead (measured medians: DESIGN.md section 3, run-time-geometry MixedNet).
BOUND_RELIED = {
    "wide": ("b0", "b1", "b2"),
    "deep": ("b0",),
    "long_stride": ("b0", "b1", "head"),
    "max_stride": ("b0", "head"),
    "stateless": ("prob",),
    "boundary": ("b0", "b1", "head"),
}
BOUND_CEILING = 0.1


@pytest.fixture(params=["ascending", "descending"])
def thread_order(request):
    """threads of a phase executed in ascending and in descending order: identical results in both rule out a
    read-after-write dependency between the threads of one phase (a missing barrier)"""
    emul.lib().emul_gen_thread_order(int(request.param == "descending"))
    yield
    emul.lib().emul_gen_thread_order(0)


def _rows(stride):
    return max(4 * stride + 20, 90)


def _ragged(g, feats, stride, int8_in=None):
    """feed feats [S, T, 40] in a ragged call sequence; row types rotate uint16 -> float32 (-> int8 for a quantised model)"""
    got = []
    cuts = call_cuts(stride, feats.shape[1])
    for i, (a, b) in enumerate(zip(cuts[:-1], cuts[1:])):
        rows = feats[:, a:b]
        if i % 3 == 1:
            rows = (rows.astype(np.float32) * R.FEATURE_SCALE).astype(np.float32)
        elif i % 3 == 2 and int8_in is not None:
            rows = R.quantize_input(rows.astype(np.float32) * R.FEATURE_SCALE, *int8_in)
        got.append(g.infer(rows))
    return np.concatenate(got, 1)


def _flat_state(m):
    return np.concatenate([np.asarray(m.st_first).ravel()] + [np.asarray(r).ravel() for r in m.st_block] + [np.asarray(m.st_head).ravel()])


def test_geometries_reach_the_edges_of_the_range():
    info = {n: emul.gen_arch_info(s.encode()) for n, s in all_geometries().items()}
    assert all(i["rc"] == 0 for i in info.values()), info
    assert info["wide"]["sm_elems"] * 4 > 48 * 1024 and info["wide"]["state_elems"] == 10846
    assert 150 * 1000 <= info["deep"]["sm_elems"] * 4 <= SMEM_CAP and GEOMETRIES["deep"].n_blocks == 8
    assert info["max_stride"]["ring0"] == 0 and info["max_stride"]["pend_cap"] == 63
    assert info["long_stride"]["pend_cap"] == 16
    assert info["stateless"]["state_elems"] == 0
    assert info["boundary"]["sm_elems"] * 4 == SMEM_CAP


def test_the_200k_boundary_pair_exists():
    """two containers whose shared memory is exactly 200 KiB and 4 bytes more (the GPU test runs the first and expects
    MWW_EUNSUPPORTED for the second)"""
    b = boundary_specs()
    assert sorted(b) == [SMEM_CAP // 4, SMEM_CAP // 4 + 1]
    for elems, spec in b.items():
        assert emul.gen_arch_info(spec.encode())["sm_elems"] == elems


@pytest.mark.parametrize("name", NAMES + ["c320"])
def test_c_oracle_equals_the_numpy_oracle(name):
    """C (oracle/mixednet.c) and NumPy (mixednet_ref.py) restatements agree at every range geometry: int8 bit for bit,
    fp32 within 1e-6.  c320 overflowed the C oracle's 256-channel step buffers; stateless has a 1-row head, whose ring the
    NumPy oracle used to grow by a row per step."""
    spec = R.Spec(64, 5, 3, (320,), ((5,),), head_rows=4) if name == "c320" else all_geometries()[name]
    f32, q8 = models(spec)
    s = spec.stride
    feats = features(1, _rows(s) * 160, 40)[0]
    n = feats.shape[0] // s * s
    x = feats[:n].astype(np.float32) * R.FEATURE_SCALE
    c_f = oracle.MixedNet(MF.write_container(f32)).predict_u16(feats)
    np_f = np.asarray(R.predict_spectrogram(R.FoldedStreamingF32(f32), feats[:n]), np.float32)
    assert c_f.shape == np_f.shape == (n // s,)
    assert np.abs(c_f - np_f).max() <= 1e-6
    m8 = R.StreamingInt8(q8)
    np_q = np.asarray(R.predict_spectrogram(m8, x, quantized=True, in_scale=m8.input_scale, in_zp=m8.input_zero_point), np.float32)
    c_q = oracle.MixedNet(MF.write_container(q8)).predict_u16(feats)
    assert np.array_equal(c_q, np_q)
    assert c_f.std() > 1e-3 and len(np.unique(c_q)) > 2                     # the comparison is not vacuous


def _refused(tensors):
    with pytest.raises(ValueError):
        oracle.MixedNet(MF.write_container(tensors))


@pytest.mark.parametrize("bad", ["channels_513", "first_conv_513", "k0_65", "stride_over_k0", "nine_blocks", "tap_65",
                                 "head_65", "stride_0"])
def test_oracles_refuse_what_they_cannot_hold(bad):
    """outside 512 channels / 64 taps / stride <= k0 / 8 blocks the C oracles return NULL (a Python error), never overflow"""
    small = R.Spec(8, 5, 3, (16,), ((3,),), head_rows=2)
    arch = {
        "channels_513": R.Spec(8, 5, 3, (513,), ((3,),), head_rows=2),
        "first_conv_513": R.Spec(513, 5, 3, (16,), ((3,),), head_rows=2),
        "k0_65": R.Spec(8, 65, 3, (16,), ((3,),), head_rows=2),
        "stride_over_k0": R.Spec(8, 5, 6, (16,), ((3,),), head_rows=2),
        "nine_blocks": R.Spec(8, 5, 3, (16,) * 9, ((3,),) * 9, head_rows=2),
        "tap_65": R.Spec(8, 5, 3, (16,), ((65,),), head_rows=2),
        "head_65": R.Spec(8, 5, 3, (16,), ((3,),), head_rows=65),
        "stride_0": R.Spec(8, 5, 0, (16,), ((3,),), head_rows=2),
    }[bad].encode()
    f32, q8 = models(small)
    for t in (f32, q8):
        t = dict(t)
        t["arch"] = arch
        _refused(t)
    # hy/mode with one (float) entry per op of the architecture it claims -- first conv, every MixConv group and 1x1 conv,
    # head -- so that only the limit checks can refuse it; the same construction on a valid architecture is accepted
    def hybrid(a):
        t = dict(f32)
        t["arch"] = a
        spec = R.Spec.decode(a)
        t["hy/mode"] = np.zeros(2 + sum(len(k) + 1 for k in spec.mixconv_kernel_sizes), np.int32)
        return MF.write_container(t)
    HR.HybridNet(hybrid(small.encode()))
    with pytest.raises(ValueError):
        HR.HybridNet(hybrid(arch))


@pytest.mark.parametrize("name", NAMES)
def test_fp32_phases_within_the_float64_bound(name, thread_order):
    """ragged calls (uint16 and float32 rows, calls with no full step, up to stride - 1 pending rows): every probability
    and every ring entry of the emulated kernel within the float64 bound, probabilities within 1e-5 of the C oracle, pending
    rows equal to the rows fed"""
    spec = all_geometries()[name]
    f32, _ = models(spec)
    s = spec.stride
    S = 3
    feats = features(S, _rows(s) * 160, 100)
    T = feats.shape[1]
    g = emul.GenF32(f32, S)
    got = _ragged(g, feats, s)
    usable = T // s * s
    assert got.shape == (S, T // s)
    want_c = np.stack([oracle.MixedNet(MF.write_container(f32)).predict_u16(feats[k, :usable]) for k in range(S)])
    assert np.abs(got - want_c).max() <= 1e-5
    assert want_c.std() > 1e-3
    bad_p = bad_r = 0
    ratios = []
    for k in range(S):
        p64, ep, vals, errs = f64_run(f32, feats[k])
        b, r = bound_violations(got[k], p64, ep)
        bad_p += b
        b, r2 = bound_violations(g.state[k], vals, errs)
        bad_r += b
        ratios += [r, r2]
    assert bad_p == 0 and bad_r == 0, "%s: %d probabilities / %d ring entries outside the float64 bound (median bound/|value| %.2e)" % (
        name, bad_p, bad_r, np.median(ratios))
    # independent of the bound: every ring entry within RING_RTOL * max(1, |v|) of the float64 value
    assert sum(ring_tolerance_violations(g.state[k], f64_run(f32, feats[k])[2]) for k in range(S)) == 0, RING_RTOL
    n_pend = T - usable
    assert g.n_pend == n_pend
    if n_pend:
        assert np.array_equal(g.pend[:, :n_pend * 40].reshape(S, n_pend, 40), feats[:, usable:].astype(np.float32) * R.FEATURE_SCALE)
    # the NumPy oracle's rings hold the same values (its own summation order: fp32 tolerance)
    m = R.FoldedStreamingF32(f32)
    R.predict_spectrogram(m, feats[0, :usable])
    assert g.state.shape[1] == _flat_state(m).size
    assert np.abs(g.state[0] - _flat_state(m)).max(initial=0) <= 1e-5


@pytest.mark.parametrize("name", NAMES)
def test_int8_phases_bit_exact(name, thread_order):
    """the same ragged calls with int8 rows as well: probabilities equal to the C oracle's, rings and pending rows equal to
    the NumPy oracle's buffers"""
    spec = all_geometries()[name]
    _, q8 = models(spec)
    s = spec.stride
    S = 3
    feats = features(S, _rows(s) * 160, 300)
    T = feats.shape[1]
    g = emul.GenI8(q8, S)
    m0 = R.StreamingInt8(q8)
    got = _ragged(g, feats, s, int8_in=(m0.input_scale, m0.input_zero_point))
    usable = T // s * s
    want = np.stack([oracle.MixedNet(MF.write_container(q8)).predict_u16(feats[k, :usable]) for k in range(S)])
    assert got.shape == want.shape == (S, T // s) and np.array_equal(got, want)
    assert len(np.unique(want)) > 2
    m = R.StreamingInt8(q8)
    R.predict_spectrogram(m, feats[0, :usable], quantized=True, in_scale=m.input_scale, in_zp=m.input_zero_point)
    assert np.array_equal(g.state[0], _flat_state(m).astype(np.int8))
    n_pend = T - usable
    assert g.n_pend == n_pend
    if n_pend:
        pend_want = R.quantize_input(feats[0, usable:].astype(np.float32) * R.FEATURE_SCALE, m.input_scale, m.input_zero_point)
        assert np.array_equal(g.pend[0, :n_pend * 40], pend_want.ravel())


@pytest.mark.parametrize("name", NAMES)
def test_the_float64_bound_is_tight_where_it_is_relied_on(name):
    """median bound / |value| of the rings listed in BOUND_RELIED stays under BOUND_CEILING, so the bound cannot become
    vacuous there without a failure"""
    f32, _ = models(all_geometries()[name])
    t = bound_tightness(f32, features(1, 48000, 4100)[0])
    loose = {k: t[k] for k in BOUND_RELIED[name] if not t[k] <= BOUND_CEILING}
    assert not loose, "%s: median bound/|value| %s (all: %s)" % (name, loose, {k: "%.1e" % v for k, v in t.items()})


def test_the_bound_catches_two_swapped_channels_across_a_thread_pass():
    """the check has teeth: with the 1x1 weights of output channels 127 and 128 of wide's first block swapped -- the last
    channel of the first pass of the 128-thread loop and the first of the second -- the emulated kernel's rings leave the
    float64 bound of the unswapped model (and its probabilities the 1e-5 tolerance of the C oracle).  The bound is a
    worst case: every layer multiplies the inherited part by sum |w|, so through three wide blocks and the head it is
    looser than 1 on a probability; on ring entries it stays within a few thousandths of the value."""
    f32, _ = models(GEOMETRIES["wide"])
    bad = dict(f32)
    w = f32["b0/pw/w"].copy()
    w[:, [127, 128]] = w[:, [128, 127]]
    bad["b0/pw/w"] = w
    feats = features(1, 90 * 160, 100)
    g = emul.GenF32(bad, 1)
    got = g.infer(feats)
    _, _, vals, errs = f64_run(f32, feats[0])
    assert bound_violations(g.state[0], vals, errs)[0] > 0
    g_ok = emul.GenF32(f32, 1)
    g_ok.infer(feats)
    assert bound_violations(g_ok.state[0], vals, errs)[0] == 0
    want = oracle.MixedNet(MF.write_container(f32)).predict_u16(feats[0])
    assert np.abs(got[0] - want).max() > 1e-3


def test_quantize_model_calibrates_a_one_row_head():
    """a model without state (1-tap blocks, 1-row head) maps each step's rows to its logit whatever came before; the int8
    logit's range is calibrated on exactly those logits"""
    spec = GEOMETRIES["stateless"]
    f32 = R.fold_bn(spec, R.init_synthetic(spec, 0))
    calib = features(1, 200 * 160, 7000)[0]
    calib = calib[: calib.shape[0] // spec.stride * spec.stride].reshape(-1, spec.stride, 40).astype(np.float32) * R.FEATURE_SCALE
    q8 = R.quantize_model(f32, calib)
    m = R.FoldedStreamingF32(f32)
    logits = [m.step(c, want_logit=True) for c in calib]
    fresh = [R.FoldedStreamingF32(f32).step(c, want_logit=True) for c in calib]
    assert logits == fresh and len(set(logits)) > 10
    scale, zp = R._act_qparams(min(logits), max(logits))
    assert np.float32(q8["q/scales"][-2]) == scale and int(q8["q/zps"][-2]) == zp
