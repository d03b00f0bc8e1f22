"""GPU side of the run-time-geometry MixedNet across the range mww_create accepts (tests/generic_range.py: 512 channels,
8 blocks with 64-tap rings, strides up to 64, a stateless model, shared memory at the 200 KiB cap): nn_generic_f32_kernel,
nn_generic_i8_kernel and nn_generic_hybrid_kernel through the C-ABI, over several waves of the grid.

  * int8: probabilities equal to the C oracle's (oracle/mixednet.c), bit for bit;
  * fp32: within 1e-5 of the C oracle; every ring entry within RING_RTOL * max(1, |v|) of the float64 value
    (mixednet_ref.StreamingF64) and, with the probabilities, inside its worst-case error bound; the rings bit-identical to
    the host emulation of the same phase functions (tests/host_emul, fmaf on both sides);
  * pending rows equal to the oracle's; streams with the same audio give identical results.

The CPU side of the same geometries is tests/test_generic_range.py."""

import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import hybrid_ref as HR
import oracle
import tflite_hybrid_writer as HW
from conftest import synth_audio
from generic_range import (GEOMETRIES, RING_RTOL, SMEM_CAP, bound_tightness, bound_violations, boundary_specs, f64_run, models,
                           ring_tolerance_violations)
from host_emul import emul
from microwakeword_b200 import _lib
from microwakeword_b200 import model_file as MF
from microwakeword_b200 import tflite_file as TF
from oracle import mixednet_ref as R

pytestmark = pytest.mark.gpu

RANGE = dict(GEOMETRIES, boundary=boundary_specs()[SMEM_CAP // 4])
MWW_EUNSUPPORTED = -5               # include/mww.h
SMEM_PER_SM = 228 * 1024            # H100: shared memory per SM; each resident CTA also reserves 1 KiB
REGS_PER_SM = 65536
N_BASE = 16                          # distinct clips; every stream adds its own noise


def _smem(spec):
    return emul.gen_arch_info(spec.encode())["sm_elems"] * 4


def _regs_per_thread(kernel):
    """registers per thread of `kernel` in the library the engine loads (cuobjdump's resource report)"""
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    out = subprocess.run([tool, "--dump-resource-usage", _lib.SO_PATH], capture_output=True, text=True, check=True).stdout
    m = re.search(r"Function \S*%s\S*:\s*REG:(\d+)" % kernel, out)
    assert m, "no resource report for %s" % kernel
    return int(m.group(1))


def _ctas_per_sm(spec, kind):
    """resident CTAs per SM of the generic kernel, computed with the occupancy calculator's rules for sm_90 from its
    register count and its shared memory (an upper figure: fewer resident CTAs would only add waves)"""
    regs = _regs_per_thread("nn_generic_f32_kernel" if kind == "f32" else "nn_generic_i8_kernel")
    regs_per_warp = (regs * 32 + 255) // 256 * 256
    by_regs = REGS_PER_SM // regs_per_warp // 4                        # 4 warps per CTA
    return max(1, min(2048 // 128, by_regs, SMEM_PER_SM // (_smem(spec) + 1024)))


def _blob(spec, kind):
    f32, q8 = models(spec)
    return MF.write_container(f32 if kind == "f32" else q8)


def _audio(torch, S, n, seed, dups):
    """int16 CUDA [S, n]: N_BASE clips, each stream with its own noise; stream d of `dups` is an exact copy of dups[d]"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    base = torch.from_numpy(np.stack([synth_audio(n, seed + i) for i in range(N_BASE)])).cuda()
    audio = base.repeat((S + N_BASE - 1) // N_BASE, 1)[:S].contiguous()
    for a in range(0, S, 2048):
        b = min(a + 2048, S)
        noisy = audio[a:b].to(torch.int32) + torch.randint(-300, 300, (b - a, n), device="cuda", generator=g, dtype=torch.int32)
        audio[a:b] = noisy.clamp(-32768, 32767).to(torch.int16)
    for d, src in dups.items():
        audio[d] = audio[src]
    return audio


def _sample(S, waves_of):
    """first and last streams and streams spread over every wave"""
    pts = [0, 1, S - 2, S - 1] + list(np.linspace(0, S - 1, 10).astype(np.int64)) + [min(waves_of * w, S - 1) for w in range(1, 4)]
    return np.unique(np.asarray(pts, np.int64))


def _check_streams(kind, spec, got, sd, feats, streams, n_pend_rows=0):
    """got [S, P] probabilities and sd the engine's state_dict after the same rows; feats uint16 [k, T, 40] are the rows of
    `streams`.  Returns (largest fp32 probability error, its bound, largest ring error / max(1, |v|)) for the report."""
    f32, q8 = models(spec)
    worst = (0.0, 0.0, 0.0)
    for k, s in enumerate(streams):
        rows = feats[k]
        T = rows.shape[0]
        usable = T // spec.stride * spec.stride
        if kind == "int8":
            want = oracle.MixedNet(MF.write_container(q8)).predict_u16(rows)
            assert np.array_equal(got[s], want), s
            g = emul.GenI8(q8, 1)
            g.infer(rows[None])
            assert np.array_equal(sd["nn"][s], g.state[0]), s
            pend = g.pend[0, :(T - usable) * 40]
        else:
            want_c = oracle.MixedNet(MF.write_container(f32)).predict_u16(rows)
            assert got.shape[1] == want_c.size and np.abs(got[s] - want_c).max(initial=0) <= 1e-5, s
            p64, ep, vals, errs = f64_run(f32, rows)
            bad_p, ratio = bound_violations(got[s], p64, ep)
            bad_r, ratio_r = bound_violations(sd["nn"][s], vals, errs)
            assert bad_p == 0 and bad_r == 0, "stream %d: %d probabilities / %d ring entries outside the float64 bound (median bound/|value| %.2e, %.2e)" % (
                s, bad_p, bad_r, ratio, ratio_r)
            # independent of the bound (a worst case that grows with depth): rings within RING_RTOL of the float64 values
            assert ring_tolerance_violations(sd["nn"][s], vals) == 0, (s, RING_RTOL)
            ring_rel = float((np.abs(sd["nn"][s] - vals) / np.maximum(1.0, np.abs(vals))).max(initial=0))
            err = np.abs(got[s] - p64)
            if err.size and err.max() > worst[0]:
                worst = (float(err.max()), float(ep[err.argmax()]), worst[2])
            worst = (worst[0], worst[1], max(worst[2], ring_rel))
            g = emul.GenF32(f32, 1)
            g.infer(rows[None])
            assert np.array_equal(sd["nn"][s], g.state[0]), s              # same phase functions, fmaf on both sides
            pend = g.pend[0, :(T - usable) * 40]
        assert sd["pending_rows"] == T - usable
        if T > usable:
            assert np.array_equal(sd["pending"][s, :T - usable].ravel(), pend), s
    return worst


@pytest.mark.parametrize("name", list(RANGE))
@pytest.mark.parametrize("kind", ["f32", "int8"])
def test_range_geometry_through_the_c_abi(torch_cuda, name, kind):
    """predict_clip on 3 s over 3 waves of the grid plus a partial one, the same audio as 480-sample step() calls, and the
    frontend's rows as ragged infer() calls of every row type: identical probabilities and state on all three paths,
    sampled streams against the oracles"""
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    spec = RANGE[name]
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    wave = sm * _ctas_per_sm(spec, kind)
    S = 3 * wave + 5
    N = 48000
    dups = {S - 3: 2, wave + 7: 5}
    audio = _audio(torch, S, N, 4100, dups)
    blob = _blob(spec, kind)
    eng = StreamEngine(blob, n_streams=S)
    assert eng.stride == spec.stride
    got = eng.predict_clip(audio).cpu().numpy()
    sd = eng.state_dict()
    for d, src in dups.items():
        assert np.array_equal(got[d], got[src]) and np.array_equal(sd["nn"][d], sd["nn"][src])
    streams = _sample(S, wave)
    feats, _ = oracle.run_pipeline(None, audio[torch.from_numpy(streams).cuda()].cpu().numpy(), want_probs=False, threads=8)
    worst = _check_streams(kind, spec, got, sd, feats, streams)
    assert got.std() > 1e-3
    report = "\n[range] %s %s: smem %d B, %d CTAs/SM (computed), %d streams, %.2f waves" % (
        name, kind, _smem(spec), _ctas_per_sm(spec, kind), S, S / wave)
    if kind == "f32":
        tight = {k: "%.1e" % v for k, v in bound_tightness(models(spec)[0], feats[0]).items()}
        report += ", largest probability error %.2e (its bound %.2e), largest ring error %.2e of max(1, |v|), median bound/|value| %s" % (
            worst[0], worst[1], worst[2], tight)
    print(report)
    # the same audio as 480-sample live steps (long_stride / max_stride: most calls run no model step)
    eng.reset()
    parts = [eng.step(audio[:, a:a + 480]) for a in range(0, N, 480)]
    stepped = torch.cat(parts, 1).cpu().numpy()
    assert stepped.shape == got.shape and np.array_equal(stepped, got)
    assert np.array_equal(eng.state_dict()["nn"], sd["nn"])
    # the frontend's rows through infer(): ragged calls of uint16 / float32 (/ int8) rows
    fe = StreamEngine(None, n_streams=S)
    rows = fe.features(audio).view(torch.int16).cpu().numpy().view(np.uint16)
    T = rows.shape[1]
    _, q8 = models(spec)
    eng.reset()
    s = spec.stride
    cuts = sorted({c for c in (0, 1, 2, s - 1, 2 * s - 1, 2 * s + 3, T // 2, T - 1, T) if 0 <= c <= T})
    out = []
    for i, (a, b) in enumerate(zip(cuts[:-1], cuts[1:])):
        r = np.ascontiguousarray(rows[:, a:b])
        if i % 3 == 1:
            r = r.astype(np.float32) * R.FEATURE_SCALE
        elif i % 3 == 2 and kind == "int8":
            r = R.quantize_input(r.astype(np.float32) * R.FEATURE_SCALE, q8["q/scales"][0], int(q8["q/zps"][0]))
        dev = torch.from_numpy(r.view(np.int16) if r.dtype == np.uint16 else r).cuda()
        out.append(eng.infer(dev.view(torch.uint16) if r.dtype == np.uint16 else dev))
    inferred = torch.cat(out, 1).cpu().numpy()
    assert np.array_equal(inferred, got)
    assert np.array_equal(eng.state_dict()["nn"], sd["nn"])


def test_wide_int8_at_65536_streams(torch_cuda):
    """65 536 streams of wide int8 (10 846 state bytes each: stream offsets past 2^29) in one 1 s call; 96 sampled
    streams bit-exact with the oracle"""
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    S, N = 65536, 16000
    spec = RANGE["wide"]
    audio = _audio(torch, S, N, 5200, {})
    eng = StreamEngine(_blob(spec, "int8"), n_streams=S)
    got = eng.predict_clip(audio).cpu().numpy()
    streams = np.unique(np.concatenate([[0, 1, S - 2, S - 1], np.linspace(0, S - 1, 94).astype(np.int64)]))
    assert streams.size == 96
    feats, _ = oracle.run_pipeline(None, audio[torch.from_numpy(streams).cuda()].cpu().numpy(), want_probs=False, threads=8)
    del audio
    sd = eng.state_dict()
    _check_streams("int8", spec, got, sd, feats, streams)


def test_deep_fp32_tiled_equals_untiled(torch_cuda):
    """deep fp32 with a scratch budget small enough for many stream tiles (non-zero `first * state_elems` offsets in
    run_nn_tile): bit-identical to the untiled engine"""
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    spec = RANGE["deep"]
    S, N = 301, 48000
    audio = _audio(torch, S, N, 6300, {})
    blob = _blob(spec, "f32")
    whole = StreamEngine(blob, n_streams=S)
    want = whole.predict_clip(audio).cpu().numpy()
    os.environ["MWW_SCRATCH_MB"] = "2"
    try:
        tiled = StreamEngine(blob, n_streams=S)
    finally:
        del os.environ["MWW_SCRATCH_MB"]
    frames = (N - 480) // 160 + 1
    assert S * frames * 40 * 2 > 3 * (2 << 20)                        # >= 2 scratch bytes per feature: at least four tiles
    assert np.array_equal(tiled.predict_clip(audio).cpu().numpy(), want)
    assert np.array_equal(tiled.state_dict()["nn"], whole.state_dict()["nn"])


def test_the_200k_boundary(torch_cuda):
    """exactly 200 KiB of shared memory runs (checked against the oracles); 4 bytes more is MWW_EUNSUPPORTED at create
    time for fp32 and int8; a hybrid container under the fp32 cap whose quantisation buffers take it over is refused at
    create time too, not at its first launch"""
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    b = boundary_specs()
    ok, over = b[SMEM_CAP // 4], b[SMEM_CAP // 4 + 1]
    assert _smem(ok) == SMEM_CAP and _smem(over) == SMEM_CAP + 4
    audio = _audio(torch, 20, 16000, 7400, {})
    streams = np.arange(20)
    feats, _ = oracle.run_pipeline(None, audio.cpu().numpy(), want_probs=False)
    for kind in ("f32", "int8"):
        eng = StreamEngine(_blob(ok, kind), n_streams=20)
        _check_streams(kind, ok, eng.predict_clip(audio).cpu().numpy(), eng.state_dict(), feats, streams)
        with pytest.raises(_lib.MwwError) as e:
            StreamEngine(_blob(over, kind), n_streams=4)
        assert e.value.code == MWW_EUNSUPPORTED
    f32, _ = models(ok)
    hy = MF.write_container(TF.tensors_from_tflite(HW.write_hybrid_mixednet(f32, lambda op, n: n >= 1024, True)))
    with pytest.raises(_lib.MwwError) as e:
        StreamEngine(hy, n_streams=4)
    assert e.value.code == MWW_EUNSUPPORTED


def test_two_handles_on_one_thread(torch_cuda):
    """wide (52 KiB) and deep (169 KiB) interleaved call by call on one thread: each launch sets its own kernel's
    shared-memory size, and both stay identical to a handle that ran alone"""
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    audio = _audio(torch, 64, 32000, 8500, {})
    engs = {n: StreamEngine(_blob(RANGE[n], "f32"), n_streams=64) for n in ("wide", "deep")}
    alone = {}
    for n in engs:
        alone[n] = engs[n].predict_clip(audio).cpu().numpy()
        engs[n].reset()
    parts = {n: [] for n in engs}
    for a in range(0, 32000, 4000):
        for n in ("wide", "deep"):
            parts[n].append(engs[n].predict_clip(audio[:, a:a + 4000].contiguous()))
    for n in engs:
        assert np.array_equal(torch.cat(parts[n], 1).cpu().numpy(), alone[n]), n


@pytest.mark.parametrize("kind", ["f32", "int8"])
def test_stateless_model(torch_cuda, kind):
    """state_elems == 0: predict_clip, step, reset(ids), state round trip and copy_nn_state on zero-byte rings; batched
    predict_spectrograms equals the per-track loop"""
    from microwakeword_b200.engine import StreamEngine
    from microwakeword_b200.inference import Model
    torch = torch_cuda
    spec = RANGE["stateless"]
    blob = _blob(spec, kind)
    audio = _audio(torch, 40, 24000, 9600, {})
    eng = StreamEngine(blob, n_streams=40)
    assert eng.state_elements == 0
    want = eng.predict_clip(audio).cpu().numpy()
    eng.reset()
    a = eng.step(audio[:, :10000].contiguous())
    sd = eng.state_dict()
    assert sd["nn"].shape == (40, 0)
    other = StreamEngine(blob, n_streams=40)
    other.load_state_dict(sd)
    rest = audio[:, 10000:].contiguous()
    b1, b2 = eng.step(rest).cpu().numpy(), other.step(rest).cpu().numpy()
    assert np.array_equal(b1, b2) and np.array_equal(np.concatenate([a.cpu().numpy(), b1], 1), want)
    eng.reset(stream_ids=[3, 17])
    assert eng.state_dict()["nn"].shape == (40, 0)
    eng.reset()
    other.reset()
    other.copy_nn_state([0, 5], eng, [3, 17])
    assert np.array_equal(eng.predict_clip(audio).cpu().numpy(), want)
    assert np.array_equal(other.predict_clip(audio).cpu().numpy(), want)
    # predict_spectrograms over tracks of uneven length == the per-track loop of one interpreter
    feats, _ = oracle.run_pipeline(None, audio[:6].cpu().numpy(), want_probs=False)
    tracks = [feats[i, : 40 + 13 * i] for i in range(6)]
    loop = Model(blob)
    per_track = [loop.predict_spectrogram(t) for t in tracks]
    batched = Model(blob).predict_spectrograms(tracks)
    assert len(batched) == len(per_track)
    for x, y in zip(batched, per_track):
        x, y = np.asarray(x, np.float32), np.asarray(y, np.float32)
        assert x.shape == y.shape and (np.array_equal(x, y) if kind == "int8" else np.abs(x - y).max(initial=0) <= 1e-6)


@pytest.mark.parametrize("name", ["wide", "deep"])
def test_int8_reset_by_id(torch_cuda, name):
    """gen_fill_state_i8_kernel: reset(ids) from host ids and from device memory (ids outside [0, S) are skipped on the
    device path and refused on the host path); reset streams then match a fresh oracle, the others carry on"""
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    spec = RANGE[name]
    S = 50
    audio = _audio(torch, S, 32000, 10700, {})
    blob = _blob(spec, "int8")
    eng = StreamEngine(blob, n_streams=S)
    eng.predict_clip(audio[:, :16000].contiguous())
    before = eng.state_dict()
    used, n_pend = eng.frontend_buffered, eng.pending_rows
    with pytest.raises(_lib.MwwError):
        eng.reset(stream_ids=[1, S])
    assert np.array_equal(eng.state_dict()["nn"], before["nn"])
    eng.reset(stream_ids=[4, 31])
    eng.reset(stream_ids=torch.tensor([-1, 9, S, 44, 1 << 30], dtype=torch.int32, device="cuda"))
    reset = [4, 9, 31, 44]
    fresh = StreamEngine(blob, n_streams=S).state_dict()
    sd = eng.state_dict()
    for s in range(S):
        assert np.array_equal(sd["nn"][s], fresh["nn"][s] if s in reset else before["nn"][s]), s
    got = eng.predict_clip(audio[:, 16000:].contiguous()).cpu().numpy()
    host = audio.cpu().numpy()
    # a reset stream starts from a fresh frontend whose buffered samples are zeros and from pending rows of real 0 (the
    # handle's counts of buffered samples and pending rows are shared by all streams)
    fresh_audio = np.concatenate([np.zeros((len(reset), used), np.int16), host[reset, 16000:]], 1)
    feats_new, _ = oracle.run_pipeline(None, fresh_audio, want_probs=False)
    for k, s in enumerate(reset):
        rows = np.concatenate([np.zeros((n_pend, 40), np.uint16), feats_new[k]])
        assert np.array_equal(got[s], oracle.MixedNet(blob).predict_u16(rows)), s
    keep = [0, 10, S - 1]
    feats_all, _ = oracle.run_pipeline(None, host[keep], want_probs=False)
    for k, s in enumerate(keep):                                     # the others: the tail of one uninterrupted run
        whole = oracle.MixedNet(blob).predict_u16(feats_all[k])
        assert np.array_equal(got[s], whole[whole.size - got.shape[1]:])


def test_hybrid_at_257_channels(torch_cuda):
    """a hybrid model (converter rule: int8 weights for ops of >= 1024 elements) with a 257-channel layer, 6 x SMs + 37
    streams through ragged calls: rings bit-identical to the hybrid oracle, probabilities within 1e-6"""
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    spec = R.Spec(64, 5, 3, (257, 96), ((5, 9), (3, 7)), head_rows=4)
    f32 = R.fold_bn(spec, R.init_synthetic(spec, 0))
    blob = MF.write_container(TF.tensors_from_tflite(HW.write_hybrid_mixednet(f32, lambda op, n: n >= 1024, True)))
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    S = 6 * sm + 37
    eng = StreamEngine(blob, n_streams=S)
    s = eng.stride
    check = np.unique(np.asarray([0, 1, sm - 1, sm, 3 * sm + 5, S - 2, S - 1]))
    ref = [HR.HybridNet(blob) for _ in check]
    pend = [np.zeros((0, 40), np.float32) for _ in check]
    rng = np.random.default_rng(12)
    for i, n in enumerate([1, 1, s - 1, s * 57 + 1, 2, s * 3, s * 20 + 2, s - 1]):
        rows = rng.integers(0, 900, (S, n, 40)).astype(np.uint16)
        rows_f = rows.astype(np.float32) * np.float32(R.FEATURE_SCALE)
        got = eng.infer(torch.from_numpy(rows_f if i % 2 else rows).cuda()).cpu().numpy()
        sd = eng.state_dict()
        for k, st in enumerate(check):
            buf = np.concatenate([pend[k], rows_f[st]])
            want = np.asarray([ref[k].step(buf[j:j + s])[0] for j in range(0, buf.shape[0] // s * s, s)], np.float32)
            pend[k] = buf[buf.shape[0] // s * s:]
            assert got.shape[1] == want.size and np.abs(got[st] - want).max(initial=0) <= 1e-6, (i, st)
            assert np.array_equal(sd["nn"][st], ref[k].state()), (i, st)
            assert sd["pending_rows"] == pend[k].shape[0]
            if pend[k].shape[0]:
                assert np.array_equal(sd["pending"][st, :pend[k].shape[0]], pend[k])
